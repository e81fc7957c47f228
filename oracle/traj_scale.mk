# Builds the reference's Trajectory time scaling for the tests (TEST INFRASTRUCTURE), like traj.mk:
# include/mpl_basis/trajectory.h, lambda.h and math.h, UNMODIFIED and compiled where they lie, behind
# ref_traj_scale_driver.cpp.  Only outputs go to _ref/ (git-ignored).  Flags mirror the reference build: -O2, no
# fast-math, no FMA contraction.  The Eigen stand-in is shim_traj/ (its 4x4 inverse() is Gauss-Jordan with partial
# pivoting, the operations of the host restatement's LambdaSeg), searched before shim/, which still supplies
# unsupported/Eigen/Polynomials.
#
#   make -C oracle -f traj_scale.mk ref
CXX ?= g++
REF_INC ?= /root/reference/include

# only where the reference sources can be read; the tests fall back to their recorded results otherwise
ref:
	@if [ -r $(REF_INC)/mpl_basis/trajectory.h ]; then \
	  $(MAKE) -f traj_scale.mk _ref/libmplref_traj_scale.so; \
	else echo "reference sources not readable under $(REF_INC): oracle/_ref/libmplref_traj_scale.so not built"; fi

_ref/libmplref_traj_scale.so: ref_traj_scale_driver.cpp ../include/mplx.h shim_traj/Eigen/Core
	mkdir -p _ref
	$(CXX) -O2 -std=c++11 -ffp-contract=off -fPIC -pthread -w -I shim_traj -I shim -I $(REF_INC) -I ../include -shared -o $@ ref_traj_scale_driver.cpp

clean:
	rm -f _ref/libmplref_traj_scale.so

.PHONY: ref clean
