"""TrajSolver for batches of paths on the device (mplx_traj_solve, include/mplx.h)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi

VEL, ACC, JRK = abi.VEL, abi.ACC, abi.JRK
SCALE, SCALE_DOWN = abi.TRAJ_SCALE, abi.TRAJ_SCALE_DOWN


def pack_paths(results, dim):
    """The waypoint slots of trajectories given as dicts with `seg_t` and `coeff` (as TrajSolverBatch.solve returns
    them): (waypoints per path, offset, seg_t, coeff) in mplx_traj_out's layout."""
    n = np.array([len(r["seg_t"]) + 1 if len(r["seg_t"]) else 0 for r in results], dtype=np.int64)
    offset = np.zeros(len(results) + 1, dtype=np.int64)
    np.cumsum(n, out=offset[1:])
    total = int(offset[-1])
    seg_t = np.zeros(max(total, 1))
    coeff = np.zeros((max(total, 1), dim + 1, 6))
    for p, r in enumerate(results):
        s = int(n[p]) - 1
        if s > 0:
            seg_t[offset[p]:offset[p] + s] = r["seg_t"]
            coeff[offset[p]:offset[p] + s] = np.asarray(r["coeff"]).reshape(s, dim + 1, 6)
    return n, offset, seg_t, coeff


def split_slots(offset, nodes, seg_t, coeff, samples=None):
    """The inverse of pack_paths for mplx_batch_traj_out's layout: one dict per path with `nodes` (the path's
    waypoint slots), `seg_t` and `coeff` (one entry per segment) and, when samples is given, `samples` (its rows)."""
    res = []
    for q in range(len(offset) - 1):
        o, o1 = int(offset[q]), int(offset[q + 1])
        s = max(o1 - o - 1, 0)
        r = dict(nodes=nodes[o:o1].copy(), seg_t=seg_t[o:o + s].copy(), coeff=coeff[o:o + s].copy())
        if samples is not None:
            r["samples"] = samples[q].copy()
        res.append(r)
    return res


def pack_lambda(scaled, offset, dim):
    """total_t, n_lambda and the lambda slots (mplx_traj_scale_out's layout) of TrajSolverBatch.scale's results
    (with_lambda=True) for the paths at `offset`."""
    NC = 5 * dim
    n_paths = len(scaled)
    total_t = np.zeros(max(n_paths, 1))
    n_lambda = np.zeros(max(n_paths, 1), dtype=np.int32)
    lam = np.zeros((max(int(offset[-1]), 1) * NC, 7))
    for p, r in enumerate(scaled):
        rows = np.asarray(r["lambda"], dtype=np.float64).reshape(-1, 7)
        total_t[p] = r["total_t"]
        n_lambda[p] = len(rows)
        lam[offset[p] * NC:offset[p] * NC + len(rows)] = rows
    return total_t, n_lambda, lam


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

    def scale(self, results, mode, mv=None, ri=1.0, rf=1.0, n_samples=0, with_lambda=False):
        """Trajectory::scale(ri, rf) (mode SCALE) or scale_down(mv, ri, rf) (SCALE_DOWN) on the device for the
        trajectories `results` (dicts with `seg_t` and `coeff`, as solve returns them).  mv, ri and rf are scalars
        or one value per path.  Returns (results, seconds): one dict per path with `status` (1: scaled; 2:
        scale_down found no velocity above mv, unchanged; 0: not scaled — fewer than 2 waypoints, a segment time
        <= 0 or not finite, a coefficient not finite, or a parameter not finite and > 0), `total_t`, `seg_T`
        (getSegmentTimes of the scaled trajectory), with with_lambda `lambda` (rows {a3, a2, a1, a0, ti, tf, dT})
        and, with n_samples > 0, `samples` = sample(n_samples) rows as solve's.

        As in the reference, sample(N)'s last time N * (total / N) can land an ulp past the last lambda segment;
        no root is then found and that row is the trajectory's start state."""
        dim = self.dim
        n_paths = len(results)
        if mode == SCALE_DOWN and mv is None:
            raise ValueError("scale_down needs mv")
        n, offset, seg_t, coeff = pack_paths(results, dim)
        total = int(offset[-1])

        def per_path(x):
            return np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (n_paths,)))

        mva = None if mv is None else per_path(mv)
        ria, rfa = per_path(ri), per_path(rf)
        NC = 5 * dim
        status = np.zeros(max(n_paths, 1), dtype=np.int32)
        total_t = np.zeros(max(n_paths, 1))
        seg_T = np.zeros(max(total, 1))
        n_lambda = np.zeros(max(n_paths, 1), dtype=np.int32)
        lam = np.zeros((max(total, 1) * NC, 7)) if with_lambda else None
        samples = np.zeros((max(n_paths, 1), n_samples + 1, 4 * dim + 3)) if n_samples > 0 else None
        out = abi.TrajScaleOut(status.ctypes.data, total_t.ctypes.data, seg_T.ctypes.data, n_lambda.ctypes.data,
                               None if lam is None else lam.ctypes.data,
                               None if samples is None else samples.ctypes.data, 0.0)
        abi.check(self._lib.mplx_traj_scale(self._h, n_paths, offset.ctypes.data, seg_t.ctypes.data, coeff.ctypes.data,
                                            mode, None if mva is None else mva.ctypes.data, ria.ctypes.data,
                                            rfa.ctypes.data, n_samples, C.byref(out)))
        res = []
        for p in range(n_paths):
            s = max(int(n[p]) - 1, 0)
            r = dict(status=int(status[p]), total_t=float(total_t[p]), seg_T=seg_T[offset[p]:offset[p] + s].copy())
            if lam is not None:
                r["lambda"] = lam[offset[p] * NC:offset[p] * NC + n_lambda[p]].copy()
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
