// ref_traj_scale_driver.cpp — the reference's UNMODIFIED Trajectory time scaling (include/mpl_basis/trajectory.h,
// lambda.h and math.h, compiled where they lie against the Eigen stand-in in shim_traj/) behind the signature of
// the product's mplh_traj_scale and mplh_solve (host/mpl_host_capi.cpp), so that the host restatement can be
// checked against it.  Trajectory::scale is called directly; scale_down, which does not compile in the reference,
// is run as the product defines it, on the reference's own classes.  TEST INFRASTRUCTURE.
// Build: make -C oracle -f traj_scale.mk ref -> oracle/_ref/libmplref_traj_scale.so (git-ignored), run by build().
#include <mpl_basis/trajectory.h>

#include <algorithm>
#include <string>

#include "mplx.h"

static thread_local std::string g_err;
extern "C" const char *mplh_last_error(void) { return g_err.c_str(); }

namespace {
// trajectory.h:173-228 does not compile (extrema_vel, Vec4f evaluate(t), i < 3 whatever Dim): its steps with the
// reference's own extrema_v, v(t), max_vel, std::sort, Lambda and Lambda::getT, over the axes i < Dim
template <int Dim>
bool scale_down(Trajectory<Dim> &traj, decimal_t mv, decimal_t ri, decimal_t rf) {
  std::vector<VirtualPoint> vs;
  VirtualPoint vi, vf;
  vi.p = ri; vi.v = 0; vi.t = 0;
  vf.p = rf; vf.v = 0; vf.t = traj.taus.back();
  vs.push_back(vi);
  for (int id = 0; id < (int)traj.segs.size(); id++) {
    for (int i = 0; i < Dim; i++) {
      if (traj.segs[id].max_vel(i) > mv) {
        std::vector<decimal_t> ts = traj.segs[id].pr(i).extrema_v(traj.segs[id].t());
        if (id != 0) ts.push_back(0);
        ts.push_back(traj.segs[id].t());
        for (const auto &tv : ts) {
          decimal_t v = traj.segs[id].pr(i).v(tv);
          decimal_t lambda_v = fabs(v) / mv;
          if (lambda_v <= 1) continue;
          VirtualPoint vt;
          vt.p = lambda_v; vt.v = 0; vt.t = tv + traj.taus[id];
          vs.push_back(vt);
        }
      }
    }
  }
  vs.push_back(vf);
  std::sort(vs.begin(), vs.end(), [](const VirtualPoint &i, const VirtualPoint &j) { return i.t < j.t; });
  decimal_t max_l = 1;
  for (const auto &v : vs)
    if (v.p > max_l) max_l = v.p;
  if (max_l <= 1) return false;
  for (int i = 1; i < (int)vs.size() - 1; i++) vs[i].p = max_l;
  std::vector<VirtualPoint> vs_s;
  vs_s.push_back(vs.front());
  for (const auto &v : vs)
    if (v.t > vs_s.back().t) vs_s.push_back(v);
  traj.lambda_ = Lambda(vs_s);
  std::vector<decimal_t> ts;
  for (const auto &tau : traj.taus) ts.push_back(traj.lambda_.getT(tau));
  traj.Ts = ts;
  traj.total_t_ = ts.back();
  return true;
}

template <int Dim>
void scale(int n_seg, const double *seg_t, const double *coeff, int control, int mode, double mv, double ri, double rf,
           int n_samples, int32_t *status, double *total_t, double *seg_T, int32_t *n_lambda, double *lambda,
           double *samples, uint8_t *flags) {
  vec_E<Primitive<Dim>> prs;
  for (int j = 0; j < n_seg; j++) {
    vec_E<Vec6f> cs(Dim + 1);
    for (int a = 0; a <= Dim; a++)
      for (int k = 0; k < 6; k++) cs[a](k) = coeff[((size_t)j * (Dim + 1) + a) * 6 + k];
    prs.push_back(Primitive<Dim>(cs, seg_t[j], (Control::Control)control));
  }
  Trajectory<Dim> traj(prs);
  const bool scaled = mode == MPLX_TRAJ_SCALE ? traj.scale(ri, rf) : scale_down<Dim>(traj, mv, ri, rf);
  *status = scaled ? 1 : 2;
  *total_t = traj.getTotalTime();
  const std::vector<decimal_t> dts = traj.getSegmentTimes();
  for (int j = 0; j < n_seg; j++) seg_T[j] = dts[j];
  seg_T[n_seg] = 0;
  const auto &ls = traj.lambda_.segs;
  if (n_lambda) *n_lambda = (int32_t)ls.size();
  if (lambda)
    for (size_t k = 0; k < ls.size(); k++) {
      double *o = lambda + k * 7;
      for (int i = 0; i < 4; i++) o[i] = ls[k].a(i);
      o[4] = ls[k].ti; o[5] = ls[k].tf; o[6] = ls[k].dT;
    }
  if (samples) {
    const auto cmds = traj.sample(n_samples);
    const int W = 4 * Dim + 3;
    for (int i = 0; i <= n_samples; i++) {
      double *o = samples + (size_t)i * W;
      for (int d = 0; d < Dim; d++) { o[d] = cmds[i].pos(d); o[Dim + d] = cmds[i].vel(d); o[2 * Dim + d] = cmds[i].acc(d); o[3 * Dim + d] = cmds[i].jrk(d); }
      o[4 * Dim] = cmds[i].yaw; o[4 * Dim + 1] = cmds[i].yaw_dot; o[4 * Dim + 2] = cmds[i].t;
    }
  }
  if (flags) {
    // 1 where Lambda::evaluate finds no segment with ti <= tau < tf for the row's tau (trajectory.h:100-110):
    // the reference then reads an uninitialised point, so the row's vel, acc and jrk are indeterminate
    const decimal_t dt = traj.getTotalTime() / n_samples;
    for (int i = 0; i <= n_samples; i++) {
      flags[i] = 0;
      if (!traj.lambda_.exist()) continue;
      decimal_t tau = traj.lambda_.getTau(i * dt);
      if (tau < 0) tau = 0;
      if (tau > traj.getTotalTime()) tau = traj.getTotalTime();
      bool found = false;
      for (const auto &seg : ls)
        if (tau >= seg.ti && tau < seg.tf) { found = true; break; }
      flags[i] = found ? 0 : 1;
    }
  }
}
}  // namespace

extern "C" {
/* mplh_traj_scale's signature (host/mpl_host_capi.cpp) plus flags[n_samples + 1]: 1 on the sample rows whose
 * lambda the reference leaves indeterminate.  Paths mplh_traj_scale gives status 0 are not scaled here either. */
int reft_traj_scale(int dim, int n_seg, const double *seg_t, const double *coeff, int control, int mode, double mv,
                    double ri, double rf, int n_samples, int32_t *status, double *total_t, double *seg_T,
                    int32_t *n_lambda, double *lambda, double *samples, uint8_t *flags) {
  if (n_seg < 1 || !seg_t || !coeff || !status || !total_t || !seg_T || (samples && n_samples < 1) ||
      (mode != MPLX_TRAJ_SCALE && mode != MPLX_TRAJ_SCALE_DOWN)) {
    g_err = "bad argument";
    return 1;
  }
  if (dim == 2) scale<2>(n_seg, seg_t, coeff, control, mode, mv, ri, rf, n_samples, status, total_t, seg_T, n_lambda, lambda, samples, flags);
  else if (dim == 3) scale<3>(n_seg, seg_t, coeff, control, mode, mv, ri, rf, n_samples, status, total_t, seg_T, n_lambda, lambda, samples, flags);
  else { g_err = "dim must be 2 or 3"; return 1; }
  return 0;
}

/* math.h's solve(a, b, c, d, e): *n roots (at most 4) into roots. */
int reft_solve(double a, double b, double c, double d, double e, int32_t *n, double *roots) {
  const std::vector<decimal_t> r = solve(a, b, c, d, e);
  *n = (int32_t)r.size();
  for (size_t k = 0; k < r.size() && k < 4; k++) roots[k] = r[k];
  return 0;
}
}
