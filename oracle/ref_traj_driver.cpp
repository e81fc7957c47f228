// ref_traj_driver.cpp — the reference's UNMODIFIED TrajSolver (include/mpl_traj_solver/traj_solver.h with
// src/mpl_traj_solver/poly_solver.cpp and poly_traj.cpp, compiled where they lie against the Eigen stand-in
// in shim_traj/) behind the signature of the product's mplh_traj_solve (host/mpl_host_capi.cpp), so that the
// host restatement can be checked against it.  TEST INFRASTRUCTURE.
// Build: make -C oracle -f traj.mk ref -> oracle/_ref/libmplref_traj.so (git-ignored), run by build().
#include <mpl_traj_solver/traj_solver.h>

#include <stdexcept>

#include "../motion_primitive_library_b200/host/traj_rows.hpp"
#include "mplx.h"

namespace {
template <int Dim>
void solve(int control, int yaw_control, const mplx_waypoint *wps, const uint8_t *wp_control, int n_wp,
           const double *dts, double v, int n_samples, int32_t *n_seg, double *seg_t, double *coeff, double *samples,
           double *waypoints) {
  TrajSolver<Dim> solver((Control::Control)control, (Control::Control)yaw_control);
  if (wp_control) {
    vec_E<Waypoint<Dim>> ws;
    for (int i = 0; i < n_wp; i++) {
      Waypoint<Dim> w((Control::Control)wp_control[i]);
      for (int d = 0; d < Dim; d++) {
        w.pos(d) = wps[i].pos[d]; w.vel(d) = wps[i].vel[d]; w.acc(d) = wps[i].acc[d]; w.jrk(d) = wps[i].jrk[d];
      }
      w.yaw = wps[i].yaw;
      ws.push_back(w);
    }
    solver.setWaypoints(ws);
  } else {
    vec_Vecf<Dim> path(n_wp);
    for (int i = 0; i < n_wp; i++)
      for (int d = 0; d < Dim; d++) path[i](d) = wps[i].pos[d];
    solver.setPath(path);
  }
  if (dts && n_wp > 0) solver.setDts(std::vector<decimal_t>(dts, dts + (n_wp - 1)));
  solver.setV(v);
  // the reference reads past the end of an empty time allocation (traj_solver.h:128-131); refuse that call
  if (n_wp >= 2 && !dts && !(v > 0)) throw std::invalid_argument("no segment times");
  const Trajectory<Dim> traj = solver.solve();
  *n_seg = (int32_t)traj.segs.size();
  const std::vector<decimal_t> used = solver.getDts();
  if (seg_t)
    for (size_t i = 0; i < used.size() && (int)i + 1 < n_wp; i++) seg_t[i] = used[i];
  if (coeff)
    for (size_t j = 0; j < traj.segs.size(); j++)
      for (int a = 0; a <= Dim; a++) {
        const Primitive1D &pr = a < Dim ? traj.segs[j].prs_[a] : traj.segs[j].pr_yaw_;
        for (int k = 0; k < 6; k++) coeff[(j * (Dim + 1) + a) * 6 + k] = pr.c(k);
      }
  if (samples) {
    const auto cmds = traj.sample(n_samples);
    for (int i = 0; i <= n_samples; i++) mplh::put_command_row<Dim>(samples, i, cmds[i]);
  }
  if (waypoints) {
    const auto ws = traj.getWaypoints();
    for (size_t i = 0; i < ws.size(); i++) mplh::put_waypoint_row<Dim>(waypoints, i, ws[i]);
  }
}
}  // namespace

extern "C" {
static thread_local std::string g_err;
const char *mplh_last_error(void) { return g_err.c_str(); }

int reft_traj_solve(int dim, int control, int yaw_control, const mplx_waypoint *wps, const uint8_t *wp_control, int n_wp,
                    const double *dts, double v, int n_samples, int32_t *n_seg, double *seg_t, double *coeff,
                    double *samples, double *waypoints) {
  if (n_wp < 0 || (n_wp > 0 && !wps) || !n_seg || (samples && n_samples < 1)) { g_err = "bad argument"; return 1; }
  *n_seg = 0;
  try {
    if (dim == 2) solve<2>(control, yaw_control, wps, wp_control, n_wp, dts, v, n_samples, n_seg, seg_t, coeff, samples, waypoints);
    else if (dim == 3) solve<3>(control, yaw_control, wps, wp_control, n_wp, dts, v, n_samples, n_seg, seg_t, coeff, samples, waypoints);
    else { g_err = "dim must be 2 or 3"; return 1; }
    return 0;
  } catch (const std::exception &e) {
    g_err = e.what();
    return 2;
  }
}
}
