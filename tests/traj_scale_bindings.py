"""Trajectory time-scaling bindings for the tests: the product's host restatement (planner.traj_scale,
planner.solve_roots) and the REFERENCE's own Trajectory::scale, scale_down steps and math.h solve
(oracle/_ref/libmplref_traj_scale.so, built by oracle/traj.mk), with the same signatures (mplh_traj_scale,
mplh_solve in host/mpl_host_capi.cpp)."""
import numpy as np

from motion_primitive_library_b200.planner import bind, run_solve, run_traj_scale, solve_roots, traj_scale  # noqa: F401
from reference_record import reference
from traj_bindings import ROOT

REF_TRAJ = ROOT / "oracle" / "_ref" / "libmplref_traj_scale.so"


def scale_reference(dim, seg_t, coeff, mode, n_samples=50, max_bytes=256, **kw):
    """The reference's scale / scale_down on one trajectory (arguments as planner.run_traj_scale), with `flags`.
    On flagged rows the reference's lambda is indeterminate, so their vel, acc and jrk are recorded as 0.  Recorded
    arrays above max_bytes are kept as digests (None: keep them all)."""
    def live():
        lib, fn = bind(REF_TRAJ, "reft_traj_scale")
        r = run_traj_scale(fn, lib, dim, seg_t, coeff, mode, n_samples=n_samples, flags=True, **kw)
        r["samples"][r["flags"] == 1, dim:4 * dim] = 0.0
        return r

    return reference(REF_TRAJ, live, max_bytes=max_bytes)


def solve_reference(a, b, c, d, e):
    """math.h's solve(a, b, c, d, e) in the reference."""
    def live():
        _, fn = bind(REF_TRAJ, "reft_solve", "mplh_solve")
        return run_solve(fn, a, b, c, d, e)

    return reference(REF_TRAJ, live, max_bytes=None)


def pv(c, t):
    """Primitive1D::v in the host's operand order (power(t, n) multiplies from 1)."""
    return c[0] / 24 * (t * t * t * t) + c[1] / 6 * (t * t * t) + c[2] / 2 * t * t + c[3] * t + c[4]


def pa(c, t):
    return c[0] / 6 * (t * t * t) + c[1] / 2 * t * t + c[2] * t + c[3]


def pj(c, t):
    return c[0] / 2 * t * t + c[1] * t + c[2]


def end_row_derivatives(dim, seg_t, coeff, lam):
    """vel, acc and jrk at the trajectory's end under the last lambda segment (the host's defined value where
    the reference's Lambda::evaluate finds no segment), in the host's operand order."""
    taus = [0.0]
    for t in seg_t:
        taus.append(float(t) + taus[-1])
    tau = taus[-1]
    a = lam[-1]
    l = a[0] * (tau * tau * tau) + a[1] * tau * tau + a[2] * tau + a[3]
    ld = 3 * a[0] * tau * tau + 2 * a[1] * tau + a[2]
    s = len(seg_t) - 1
    t = tau - taus[s]
    out = np.zeros(3 * dim)
    for k in range(dim):
        c = coeff[s, k]
        vel = pv(c, t) / l
        acc = pa(c, t) / l / l - vel * ld / l / l / l
        out[k] = vel
        out[dim + k] = acc
        out[2 * dim + k] = pj(c, t) / l / l - 3 / (l * l * l) * acc * acc * ld + 3 / (l * l * l * l) * vel * ld * ld
    return out
