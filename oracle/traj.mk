# Builds the reference's trajectory code for the tests (TEST INFRASTRUCTURE), like the `ref` target of
# oracle/Makefile: UNMODIFIED reference sources compiled where they lie, each behind its driver.  Only outputs go
# to _ref/ (git-ignored).  Flags mirror the reference build: -O2, no fast-math, no FMA contraction.
#
#   _ref/libmplref_traj.so        the trajectory solver: include/mpl_traj_solver/traj_solver.h with
#                                 src/mpl_traj_solver/poly_solver.cpp and poly_traj.cpp, behind ref_traj_driver.cpp
#   _ref/libmplref_traj_scale.so  Trajectory's time scaling: include/mpl_basis/trajectory.h, lambda.h and math.h,
#                                 behind ref_traj_scale_driver.cpp
#   _ref/libmplref_traj_check.so  the trajectory checks: include/mpl_planner/env/env_map.h (traverse_trajectory,
#                                 is_free), include/mpl_basis/primitive.h (validate_primitive), trajectory.h and
#                                 lambda.h, behind ref_traj_check_driver.cpp
#
# The Eigen stand-in is shim_traj/ (dense dynamic-size algebra added to shim/'s), searched before shim/, which
# still supplies Boost and unsupported/Eigen/Polynomials.  This pins the reference's algorithms under the
# stand-in's dense algebra — products summed in increasing k, Doolittle LU with row partial pivoting, a 4x4
# inverse() by Gauss-Jordan with partial pivoting: the operations of the host restatement
# (motion_primitive_library_b200/host/mpl_host.hpp) — not under Eigen's blocked LU and GEMM, whose rounding can
# differ in the last bits.
#
#   make -C oracle -f traj.mk ref
CXX ?= g++
REF_INC ?= /root/reference/include
REF_FLAGS = -O2 -std=c++11 -ffp-contract=off -fPIC -pthread -w -I shim_traj -I shim -I $(REF_INC) -I ../include -shared

# each library only where its reference header can be read; the tests fall back to their recorded results otherwise
ref:
	@for x in "libmplref_traj.so mpl_traj_solver/traj_solver.h" "libmplref_traj_scale.so mpl_basis/trajectory.h" \
	          "libmplref_traj_check.so mpl_planner/env/env_map.h"; do \
	  set -- $$x; \
	  if [ -r $(REF_INC)/$$2 ]; then $(MAKE) -f traj.mk _ref/$$1 || exit 1; \
	  else echo "reference sources not readable under $(REF_INC): oracle/_ref/$$1 not built"; fi; \
	done

_ref/libmplref_traj.so: ref_traj_driver.cpp ../include/mplx.h ../motion_primitive_library_b200/host/traj_rows.hpp shim_traj/Eigen/Core
	mkdir -p _ref
	$(CXX) $(REF_FLAGS) -o $@ ref_traj_driver.cpp $(REF_INC)/../src/mpl_traj_solver/poly_solver.cpp $(REF_INC)/../src/mpl_traj_solver/poly_traj.cpp

_ref/libmplref_traj_scale.so: ref_traj_scale_driver.cpp ../include/mplx.h ../motion_primitive_library_b200/host/traj_rows.hpp shim_traj/Eigen/Core
	mkdir -p _ref
	$(CXX) $(REF_FLAGS) -o $@ ref_traj_scale_driver.cpp

_ref/libmplref_traj_check.so: ref_traj_check_driver.cpp ../include/mplx.h shim_traj/Eigen/Core shim/Eigen/Core
	mkdir -p _ref
	$(CXX) $(REF_FLAGS) -o $@ ref_traj_check_driver.cpp

clean:
	rm -f _ref/libmplref_traj.so _ref/libmplref_traj_scale.so _ref/libmplref_traj_check.so

.PHONY: ref clean
