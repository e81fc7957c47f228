# Builds the reference's trajectory solver for the tests (TEST INFRASTRUCTURE), like the `ref` target of
# oracle/Makefile: include/mpl_traj_solver/traj_solver.h with src/mpl_traj_solver/poly_solver.cpp and
# poly_traj.cpp, UNMODIFIED and compiled where they lie, behind ref_traj_driver.cpp.  Only outputs go to _ref/
# (git-ignored).  Flags mirror the reference build: -O2, no fast-math, no FMA contraction.
#
# The Eigen stand-in is shim_traj/ (dense dynamic-size algebra added to shim/'s), searched before shim/, which
# still supplies Boost and unsupported/.  This pins the reference's algorithm under the stand-in's dense
# algebra — products summed in increasing k, Doolittle LU with row partial pivoting, the same operations as
# the host restatement (motion_primitive_library_b200/host/mpl_host.hpp) — not under Eigen's blocked LU and
# GEMM, whose rounding can differ in the last bits.
#
#   make -C oracle -f traj.mk ref
CXX ?= g++
REF_INC ?= /root/reference/include

# only where the reference sources can be read; the tests fall back to their recorded results otherwise
ref:
	@if [ -r $(REF_INC)/mpl_traj_solver/traj_solver.h ]; then \
	  $(MAKE) -f traj.mk _ref/libmplref_traj.so; \
	else echo "reference sources not readable under $(REF_INC): oracle/_ref/libmplref_traj.so not built"; fi

_ref/libmplref_traj.so: ref_traj_driver.cpp ../include/mplx.h shim_traj/Eigen/Core
	mkdir -p _ref
	$(CXX) -O2 -std=c++11 -ffp-contract=off -fPIC -pthread -w -I shim_traj -I shim -I $(REF_INC) -I ../include -shared -o $@ ref_traj_driver.cpp $(REF_INC)/../src/mpl_traj_solver/poly_solver.cpp $(REF_INC)/../src/mpl_traj_solver/poly_traj.cpp

clean:
	rm -f _ref/libmplref_traj.so

.PHONY: ref clean
