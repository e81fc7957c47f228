"""TrajSolver bindings for the tests: the product's host restatement (planner.traj_solve) and the REFERENCE's
own TrajSolver (oracle/_ref/libmplref_traj.so, built by oracle/traj.mk: src/mpl_traj_solver compiled against
oracle/shim_traj), with the same signature (mplh_traj_solve, host/mpl_host_capi.cpp)."""
from pathlib import Path

from motion_primitive_library_b200.planner import bind, run_traj_solve, traj_solve  # noqa: F401
from reference_record import reference

ROOT = Path(__file__).resolve().parent.parent
REF_TRAJ = ROOT / "oracle" / "_ref" / "libmplref_traj.so"


def traj_reference(dim, control, max_bytes=256, **kw):
    """The reference's TrajSolver<dim> on one path (arguments as planner.run_traj_solve).  Recorded arrays above
    max_bytes are kept as digests (None: keep them all)."""
    def live():
        lib, fn = bind(REF_TRAJ, "reft_traj_solve", "mplh_traj_solve")
        return run_traj_solve(fn, lib, dim, control, **kw)

    return reference(REF_TRAJ, live, max_bytes=max_bytes)
