# Builds the reference's trajectory checks for the tests (TEST INFRASTRUCTURE), like traj_scale.mk:
# include/mpl_planner/env/env_map.h (traverse_trajectory, is_free), include/mpl_basis/primitive.h
# (validate_primitive), trajectory.h and lambda.h, UNMODIFIED and compiled where they lie, behind
# ref_traj_check_driver.cpp.  Only outputs go to _ref/ (git-ignored).  Flags mirror the reference build: -O2, no
# fast-math, no FMA contraction.  shim_traj/ is searched before shim/, which supplies Boost and
# unsupported/Eigen/Polynomials.
#
#   make -C oracle -f traj_check.mk ref
CXX ?= g++
REF_INC ?= /root/reference/include

# only where the reference sources can be read; the tests fall back to their recorded results otherwise
ref:
	@if [ -r $(REF_INC)/mpl_planner/env/env_map.h ]; then \
	  $(MAKE) -f traj_check.mk _ref/libmplref_traj_check.so; \
	else echo "reference sources not readable under $(REF_INC): oracle/_ref/libmplref_traj_check.so not built"; fi

_ref/libmplref_traj_check.so: ref_traj_check_driver.cpp ../include/mplx.h shim_traj/Eigen/Core shim/Eigen/Core
	mkdir -p _ref
	$(CXX) -O2 -std=c++11 -ffp-contract=off -fPIC -pthread -w -I shim_traj -I shim -I $(REF_INC) -I ../include -shared -o $@ ref_traj_check_driver.cpp

clean:
	rm -f _ref/libmplref_traj_check.so

.PHONY: ref clean
