"""TrajSolver for batches of paths on the device (mplx_traj_solve, include/mplx.h)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi

VEL, ACC, JRK = abi.VEL, abi.ACC, abi.JRK


class TrajSolverBatch:
    """Smooth many paths at once: for each path, the piecewise polynomial through its waypoints that minimises the
    integral of the squared velocity (control VEL), acceleration (ACC) or jerk (JRK), as TrajSolver<dim> gives it,
    with the yaw axis from its own pass (yaw_control).  Owns a libmplx ctx on `device`; its scratch is kept
    between calls."""

    def __init__(self, dim: int, device: int = 0):
        self._lib = abi.load()
        self.dim = dim
        h = C.c_void_p()
        abi.check(self._lib.mplx_create(dim, device, C.byref(h)))
        self._h = h

    def solve(self, paths, control, yaw_control=VEL, dts=None, v=1.0, wp_control=None, n_samples=0):
        """paths: a list of waypoint arrays, one per path — (n, dim) positions (setPath; wp_control None) or
        abi.WAYPOINT_DTYPE arrays with wp_control a list of per-waypoint control-flag arrays (setWaypoints).
        dts: None (segment times |p_j+1 - p_j|_inf / v) or a list of (n - 1,) arrays.  Returns (results, seconds):
        one dict per path with `status` (1: solved, finite), `seg_t` (n - 1,), `coeff` (n - 1, dim + 1, 6:
        Primitive1D coefficients, highest order first, axes then yaw) and, with n_samples > 0, `samples`
        (n_samples + 1, 4 dim + 3) = Trajectory::sample(n_samples) rows {pos, vel, acc, jrk, yaw, yaw_dot, t};
        seconds is the device time of the kernels."""
        dim = self.dim
        n = np.array([len(p) for p in paths], dtype=np.int64)
        offset = np.zeros(len(paths) + 1, dtype=np.int64)
        np.cumsum(n, out=offset[1:])
        total = int(offset[-1])
        wps = np.zeros(max(total, 1), dtype=abi.WAYPOINT_DTYPE)
        ctl = None
        for p, path in enumerate(paths):
            sl = slice(offset[p], offset[p + 1])
            if wp_control is None:
                wps["pos"][sl, :dim] = np.asarray(path, dtype=np.float64).reshape(-1, dim)
            else:
                wps[sl] = np.asarray(path, dtype=abi.WAYPOINT_DTYPE)
        if wp_control is not None:
            ctl = np.zeros(max(total, 1), dtype=np.uint8)
            for p, c in enumerate(wp_control):
                ctl[offset[p]:offset[p + 1]] = c
        d = None
        if dts is not None:
            d = np.zeros(max(total, 1))
            for p, t in enumerate(dts):
                d[offset[p]:offset[p] + max(n[p] - 1, 0)] = t
        status = np.zeros(max(len(paths), 1), dtype=np.int32)
        seg_t = np.zeros(max(total, 1))
        coeff = np.zeros((max(total, 1), dim + 1, 6))
        samples = np.zeros((max(len(paths), 1), n_samples + 1, 4 * dim + 3)) if n_samples > 0 else None
        out = abi.TrajOut(status.ctypes.data, seg_t.ctypes.data, coeff.ctypes.data,
                          None if samples is None else samples.ctypes.data, 0.0)
        abi.check(self._lib.mplx_traj_solve(self._h, len(paths), offset.ctypes.data, wps.ctypes.data,
                                            None if ctl is None else ctl.ctypes.data,
                                            None if d is None else d.ctypes.data, float(v), control, yaw_control,
                                            n_samples, C.byref(out)))
        res = []
        for p in range(len(paths)):
            s = max(int(n[p]) - 1, 0)
            r = dict(status=int(status[p]), seg_t=seg_t[offset[p]:offset[p] + s].copy(),
                     coeff=coeff[offset[p]:offset[p] + s].copy())
            if samples is not None:
                r["samples"] = samples[p].copy()
            res.append(r)
        return res, out.seconds

    def launch_count(self) -> int:
        return int(self._lib.mplx_launch_count(self._h))

    def close(self):
        if self._h:
            self._lib.mplx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
