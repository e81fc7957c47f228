"""The block-tridiagonal statement of TrajSolver (traj_restatement.py) against the host's dense restatement
(MPL::TrajSolver, mpl_host.hpp) on random paths: both sampled by the host Trajectory, within 1e-9 relative."""
import numpy as np
import pytest

import traj_restatement as TR
from motion_primitive_library_b200 import planner as P

CONTROLS = [0x01, 0x03, 0x07, 0x11, 0x13, 0x17]


def random_waypoints(rng, dim, n, h):
    w = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
    w["pos"][:, :dim] = rng.uniform(-5, 5, (n, dim))
    w["vel"][:, :dim] = rng.uniform(-1, 1, (n, dim))
    w["acc"][:, :dim] = rng.uniform(-1, 1, (n, dim))
    w["yaw"] = rng.uniform(-1, 1, n)
    ctl = rng.choice([0x01, 0x03, 0x07, 0x13], n).astype(np.uint8)
    ctl[[0, -1]] = rng.choice([0x03, 0x07], 2)
    return w, ctl


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("yaw_control", [0x01, 0x03, 0x07])
def test_restatement_matches_host(dim, control, yaw_control):
    rng = np.random.default_rng(dim * 1000 + control * 10 + yaw_control)
    for trial in range(4):
        n = int(rng.integers(2, 40))
        kw = dict(yaw_control=yaw_control)
        if trial % 2 == 0:
            kw.update(pos=rng.uniform(-5, 5, (n, dim)), v=float(rng.uniform(0.5, 2)))
        else:
            w, ctl = random_waypoints(rng, dim, n, TR.ORDER[control])
            kw.update(waypoints=w, wp_control=ctl, dts=rng.uniform(0.05, 5, n - 1))
        host = P.traj_solve(dim, control, n_samples=64, **kw)
        mine = TR.traj_solve(dim, control, **kw)
        assert mine["status"] == 1 and host["segments"] == n - 1
        np.testing.assert_array_equal(mine["seg_t"], host["seg_t"])
        ctl0 = control if "pos" in kw else int(kw["wp_control"][0])
        s, w = P.traj_sample(dim, mine["seg_t"], mine["coeff"], ctl0, 64)
        TR.assert_close(s, host["samples"], dim, what=(n, trial))
        TR.assert_close(w, host["waypoints"], dim, what=(n, trial))
