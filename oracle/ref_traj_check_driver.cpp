// ref_traj_check_driver.cpp — the reference's UNMODIFIED trajectory checks (env_map::traverse_trajectory and
// env_map::is_free in include/mpl_planner/env/env_map.h, validate_primitive in include/mpl_basis/primitive.h, on
// its own Trajectory and Lambda, compiled where they lie against the Eigen stand-ins in shim_traj/ and shim/)
// behind the signature of the product's mplh_traj_check (host/mpl_host_capi.cpp), so that the host restatement
// can be checked against it.  A scaled path gets its lambda segments and total time assigned to the reference's
// Trajectory members.  Paths and segments where the reference is undefined (mplh_traj_check's status 0, a sample
// count above MPLX_SAMPLE_N_MAX) are not evaluated.  TEST INFRASTRUCTURE.
// Build: make -C oracle -f traj.mk ref -> oracle/_ref/libmplref_traj_check.so (git-ignored), run by build().
#include <mpl_basis/trajectory.h>
#include <mpl_planner/env/env_map.h>

#include <cmath>
#include <string>

#include "mplx.h"

static thread_local std::string g_err;
extern "C" const char *mplh_last_error(void) { return g_err.c_str(); }

namespace {
template <int Dim>
void check(const int8_t *map, const int32_t *mdim, const double *origin, double res, const int8_t *potential,
           double potential_weight, double gradient_weight, const uint8_t *region, double v_max, double a_max,
           double j_max, double yaw_max, int n_paths, const int64_t *offset, const double *seg_t, const double *coeff,
           const uint8_t *control, const double *total_t, const int32_t *n_lambda, const double *lambda,
           int32_t *status, double *cost, uint8_t *seg_free, uint8_t *seg_valid) {
  std::shared_ptr<MPL::MapUtil<Dim>> mu(new MPL::MapUtil<Dim>);
  Vecf<Dim> ori;
  Veci<Dim> md;
  size_t nvox = 1;
  for (int k = 0; k < Dim; k++) {
    ori(k) = origin[k];
    md(k) = mdim[k];
    nvox *= (size_t)mdim[k];
  }
  mu->setMap(ori, md, MPL::Tmap(map, map + nvox), res);
  MPL::env_map<Dim> env(mu);
  env.set_v_max(v_max);
  env.set_a_max(a_max);
  env.set_j_max(j_max);
  env.set_yaw_max(yaw_max);
  if (potential) {
    env.set_potential_map(std::vector<int8_t>(potential, potential + nvox));
    env.set_potential_weight(potential_weight);
    env.set_gradient_weight(gradient_weight);
  }
  if (region) {
    std::vector<bool> r(nvox);
    for (size_t i = 0; i < nvox; i++) r[i] = region[i] != 0;
    env.set_search_region(r);
  }
  for (int p = 0; p < n_paths; p++) {
    const int64_t b = offset[p];
    const int S = (int)(offset[p + 1] - b) - 1;
    status[p] = 0;
    cost[p] = 0;
    for (int j = 0; j <= S; j++) {
      if (seg_free) seg_free[b + j] = 0;
      if (seg_valid) seg_valid[b + j] = 0;
    }
    bool ok = S >= 1;
    for (int j = 0; ok && j < S; j++) ok = std::isfinite(seg_t[b + j]) && seg_t[b + j] > 0;
    for (size_t k = 0; ok && k < (size_t)S * (Dim + 1) * 6; k++) ok = std::isfinite(coeff[(size_t)b * (Dim + 1) * 6 + k]);
    if (!ok) continue;
    vec_E<Primitive<Dim>> prs;
    for (int j = 0; j < S; j++) {
      vec_E<Vec6f> cs(Dim + 1);
      for (int a = 0; a <= Dim; a++)
        for (int k = 0; k < 6; k++) cs[a](k) = coeff[((size_t)(b + j) * (Dim + 1) + a) * 6 + k];
      prs.push_back(Primitive<Dim>(cs, seg_t[b + j], (Control::Control)(control ? control[p] : 0)));
    }
    Trajectory<Dim> traj(prs);
    if (lambda && n_lambda[p] > 0) {
      for (int k = 0; k < n_lambda[p]; k++) {
        const double *r = lambda + ((size_t)b * 5 * Dim + k) * 7;
        LambdaSeg g;
        for (int i = 0; i < 4; i++) g.a(i) = r[i];
        g.ti = r[4]; g.tf = r[5]; g.dT = r[6];
        traj.lambda_.segs.push_back(g);
      }
      traj.total_t_ = total_t[p];
    }
    const double nd = std::ceil(v_max * traj.getTotalTime() / res);
    if (nd >= 1 && nd <= MPLX_SAMPLE_N_MAX) {
      status[p] = 1;
      cost[p] = env.traverse_trajectory(traj);
    }
    for (int j = 0; j < S; j++) {
      const Primitive<Dim> &pr = traj.segs[j];
      if (seg_free) {
        decimal_t max_v = 0;
        for (int i = 0; i < Dim; i++)
          if (pr.max_vel(i) > max_v) max_v = pr.max_vel(i);
        seg_free[b + j] = std::ceil(max_v * pr.t() / res) <= MPLX_SAMPLE_N_MAX && env.is_free(pr) ? 1 : 0;
      }
      if (seg_valid) seg_valid[b + j] = validate_primitive(pr, v_max, a_max, j_max, yaw_max) ? 1 : 0;
    }
  }
}
}  // namespace

extern "C" {
/* mplh_traj_check's signature (host/mpl_host_capi.cpp); nthreads is ignored (one thread). */
int reft_traj_check(int dim, const int8_t *map, const int32_t *mdim, const double *origin, double res,
                    const int8_t *potential, double potential_weight, double gradient_weight, const uint8_t *region,
                    double v_max, double a_max, double j_max, double yaw_max, int n_paths, const int64_t *offset,
                    const double *seg_t, const double *coeff, const uint8_t *control, const double *total_t,
                    const int32_t *n_lambda, const double *lambda, int nthreads, int32_t *status, double *cost,
                    uint8_t *seg_free, uint8_t *seg_valid) {
  (void)nthreads;
  if (!map || !mdim || !origin || n_paths < 0 || !offset || !status || !cost || (seg_valid && !control) ||
      (lambda && (!n_lambda || !total_t))) {
    g_err = "bad argument";
    return 1;
  }
  if (dim == 2) check<2>(map, mdim, origin, res, potential, potential_weight, gradient_weight, region, v_max, a_max, j_max, yaw_max, n_paths, offset, seg_t, coeff, control, total_t, n_lambda, lambda, status, cost, seg_free, seg_valid);
  else if (dim == 3) check<3>(map, mdim, origin, res, potential, potential_weight, gradient_weight, region, v_max, a_max, j_max, yaw_max, n_paths, offset, seg_t, coeff, control, total_t, n_lambda, lambda, status, cost, seg_free, seg_valid);
  else { g_err = "dim must be 2 or 3"; return 1; }
  return 0;
}
}
