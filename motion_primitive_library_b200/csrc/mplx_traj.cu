// mplx_traj.cu — TrajSolver for batches of paths (mplx_traj_solve, include/mplx.h), their time scaling
// (mplx_traj_scale) and their checks against the map and the dynamic limits (mplx_traj_check).
//
// The reference (src/mpl_traj_solver/poly_solver.cpp) assembles dense (S*N) x (S*N) matrices for a path of S
// segments and LU-factors them.  Here each path is solved in O(S): the cost of segment i in the derivatives at
// its two end waypoints is H_i = tau^(1-2R) * Sc * Hbar * Sc, Sc = diag(tau^k), with Hbar a constant 2h x 2h
// matrix per order (h = N/2 = R), so the system in the free derivatives is block-tridiagonal in waypoint order
// with h x h blocks.  Fixed derivatives take a unit row and column, which keeps every block h x h; one block
// Cholesky sweep per path solves it.
//   traj_sweep_kernel   one thread per path: segment times, the running sum of them, the sweep (axes, then yaw)
//   traj_coeff_kernel   one thread per segment: Primitive1D coefficients from the end-point derivatives
//   traj_sample_kernel  one thread per sample: Trajectory::sample(N) of those coefficients, in the host's
//                       operand order (include/mpl_basis/trajectory.h:100-137, primitive.h:128-145)
#include <algorithm>

#include "mplx_dispatch.h"
#include "mplx_internal.h"

namespace mplx {
namespace {

// The refusals the three batch calls share, in the order they make them.  arrays: offset and the call's other
// required arrays are given; wp_in: its per-waypoint inputs are given, which may be NULL when no path has a
// waypoint slot; samples: it is asked for n_samples + 1 sample rows per path.  Sets n_wp = offset[n_paths].
int check_batch(int n_paths, const int64_t *offset, bool arrays, bool wp_in, bool samples, int n_samples,
                long long &n_wp) {
  if (n_paths < 0) return fail(MPLX_ERR_ARG, "n_paths < 0");
  if (!offset || !arrays) return fail(MPLX_ERR_ARG, "missing array");
  if (samples && n_samples <= 0) return fail(MPLX_ERR_ARG, "samples with n_samples <= 0");
  if (offset[0] != 0) return fail(MPLX_ERR_ARG, "offset[0] must be 0");
  for (int p = 0; p < n_paths; p++)
    if (offset[p + 1] < offset[p]) return fail(MPLX_ERR_ARG, "offset decreases at path %d", p);
  n_wp = offset[n_paths];
  if (n_wp > 0 && !wp_in) return fail(MPLX_ERR_ARG, "missing array");
  if (samples && (long long)n_paths * (n_samples + 1) >= ((long long)1 << 40)) return fail(MPLX_ERR_ARG, "too many samples");
  return MPLX_OK;
}

// Launches k over n items in blocks of 128 threads, at least one: one thread per item, or, for a grid-stride
// kernel (stride), at most 16 blocks per SM.  Counts the launch once it is made.
template <class... P, class... A>
cudaError_t launch(void (*k)(P...), long long n, bool stride, cudaStream_t st, int *launches, const A &...args) {
  long long blocks = (n + 127) / 128;
  if (stride) blocks = std::min<long long>(blocks, (long long)sm_count() * 16);
  k<<<(int)std::max<long long>(blocks, 1), 128, 0, st>>>(args...);
  if (cudaError_t e = cudaGetLastError()) return e;
  *launches += 1;
  return cudaSuccess;
}

// Hbar for h = 1, 2, 3: the cost of a unit-duration segment in [start derivatives (h), end derivatives (h)]
__constant__ double kHbar1[4] = {1, -1, -1, 1};
__constant__ double kHbar2[16] = {12, 6, -12, 6, 6, 4, -6, 2, -12, -6, 12, -6, 6, 2, -6, 4};
__constant__ double kHbar3[36] = {720,  360,  60,  -720, 360,  -60, 360,  192, 36, -360, 168, -24,
                                  60,   36,   9,   -60,  24,   -3,  -720, -360, -60, 720, -360, 60,
                                  360,  168,  24,  -360, 192,  -36, -60,  -24, -3, 60,   -36,  9};
// inverse of B(k, m) = (h+m)! / (h+m-k)!: the top h coefficients (scaled by tau^(h+m)) from the end derivatives
__constant__ double kBinv2[4] = {3, -1, -2, 1};
__constant__ double kBinv3[9] = {10, -4, 0.5, -15, 7, -1, 6, -3, 0.5};

template <int H>
__device__ __forceinline__ double hbar(int a, int b) {
  if (H == 1) return kHbar1[a * 2 + b];
  if (H == 2) return kHbar2[a * 4 + b];
  return kHbar3[a * 6 + b];
}
template <int H>
__device__ __forceinline__ double binv(int a, int b) {
  if (H == 1) return 1.0;
  if (H == 2) return kBinv2[a * 2 + b];
  return kBinv3[a * 3 + b];
}

// Which derivatives of waypoint j are fixed and their values, for the axes pass (YAW false) or the yaw pass.
struct PathIn {
  const mplx_waypoint *w;  // the path's waypoints
  const uint8_t *ctl;      // per-waypoint control (setWaypoints), or NULL (setPath)
  int end_ctl;             // the endpoints' control: `control` (axes, setPath) or `yaw_control` (yaw)
  int W;
  bool yaw;
  __device__ int flags(int j, int H) const {
    const bool end = j == 0 || j == W - 1;
    const int c = (!yaw && ctl) ? ctl[j] : (end ? end_ctl : MPLX_VEL);
    return c & ((1 << H) - 1);  // use_pos, use_vel, use_acc: bit k fixes derivative k
  }
  __device__ double val(int j, int k, int a) const {
    if (yaw) return (k == 0 && ctl) ? w[j].yaw : 0.0;
    if (k == 0) return w[j].pos[a];
    if (!ctl) return 0.0;
    return k == 1 ? w[j].vel[a] : w[j].acc[a];
  }
};

// The blocks of H_i for duration tau: ss = [start, start], se = [start, end], ee = [end, end].
template <int H>
__device__ __forceinline__ void seg_blocks(double tau, double (&ss)[H][H], double (&se)[H][H], double (&ee)[H][H]) {
  double tp[H];
  tp[0] = 1.0;
#pragma unroll
  for (int k = 1; k < H; k++) tp[k] = tp[k - 1] * tau;
  double t2r = tau;  // tau^(2R-1)
#pragma unroll
  for (int k = 1; k < 2 * H - 1; k++) t2r *= tau;
#pragma unroll
  for (int a = 0; a < H; a++)
#pragma unroll
    for (int b = 0; b < H; b++) {
      const double s = tp[a] * tp[b] / t2r;
      ss[a][b] = hbar<H>(a, b) * s;
      se[a][b] = hbar<H>(a, H + b) * s;
      ee[a][b] = hbar<H>(H + a, H + b) * s;
    }
}

// Cholesky factor of an SPD H x H matrix, lower triangle packed row by row (H(H+1)/2 <= 6 entries).
template <int H>
__device__ __forceinline__ void chol(const double (&K)[H][H], double (&L)[6]) {
#pragma unroll
  for (int i = 0; i < H; i++)
#pragma unroll
    for (int j = 0; j <= i; j++) {
      double s = K[i][j];
#pragma unroll
      for (int k = 0; k < j; k++) s -= L[i * (i + 1) / 2 + k] * L[j * (j + 1) / 2 + k];
      L[i * (i + 1) / 2 + j] = i == j ? sqrt(s) : s / L[j * (j + 1) / 2 + j];
    }
}
// x := (L L^T)^-1 x
template <int H>
__device__ __forceinline__ void chol_solve(const double (&L)[6], double (&x)[H]) {
#pragma unroll
  for (int i = 0; i < H; i++) {
#pragma unroll
    for (int k = 0; k < i; k++) x[i] -= L[i * (i + 1) / 2 + k] * x[k];
    x[i] /= L[i * (i + 1) / 2 + i];
  }
#pragma unroll
  for (int i = H - 1; i >= 0; i--) {
#pragma unroll
    for (int k = i + 1; k < H; k++) x[i] -= L[k * (k + 1) / 2 + i] * x[k];
    x[i] /= L[i * (i + 1) / 2 + i];
  }
}

// Minimises sum_i d_i^T H_i d_i over the free derivatives of one path (W >= 2) for NC columns (axes) and writes
// every waypoint's derivatives to D[j*H*NC + k*NC + a]; fac holds W packed Cholesky factors.  Two waypoints
// solve nothing: their free derivatives are 0 (PolySolver, poly_solver.cpp:205).
template <int H, int NC>
__device__ void sweep(const PathIn &in, const double *seg_t, double *fac, double *D) {
  const int W = in.W;
  constexpr int HN = H * NC;
  if (W > 2) {
    double yp[H][NC], Lp[6], sep[H][H], eep[H][H];
    int fmp = 0;
    for (int j = 0; j < W; j++) {
      const int fm = in.flags(j, H);
      double K[H][H], b[H][NC], ss[H][H], se[H][H], ee[H][H];
#pragma unroll
      for (int r = 0; r < H; r++) {
#pragma unroll
        for (int c = 0; c < H; c++) K[r][c] = j > 0 ? eep[r][c] : 0.0;
#pragma unroll
        for (int a = 0; a < NC; a++) b[r][a] = 0.0;
      }
      if (j < W - 1) {
        seg_blocks<H>(seg_t[j], ss, se, ee);
#pragma unroll
        for (int r = 0; r < H; r++)
#pragma unroll
          for (int c = 0; c < H; c++) K[r][c] += ss[r][c];
      }
      // right-hand side: what the fixed derivatives of waypoints j-1, j, j+1 contribute to the free rows
      const int fmn = j < W - 1 ? in.flags(j + 1, H) : 0;
#pragma unroll
      for (int c = 0; c < H; c++)
#pragma unroll
        for (int a = 0; a < NC; a++) {
          if ((fm >> c) & 1) {
            const double f = in.val(j, c, a);
#pragma unroll
            for (int r = 0; r < H; r++) b[r][a] -= K[r][c] * f;
          }
          if (j > 0 && ((fmp >> c) & 1)) {
            const double f = in.val(j - 1, c, a);
#pragma unroll
            for (int r = 0; r < H; r++) b[r][a] -= sep[c][r] * f;
          }
          if (j < W - 1 && ((fmn >> c) & 1)) {
            const double f = in.val(j + 1, c, a);
#pragma unroll
            for (int r = 0; r < H; r++) b[r][a] -= se[r][c] * f;
          }
        }
      // fixed rows and columns become unit ones
#pragma unroll
      for (int r = 0; r < H; r++)
        if ((fm >> r) & 1) {
#pragma unroll
          for (int c = 0; c < H; c++) K[r][c] = K[c][r] = 0.0;
          K[r][r] = 1.0;
#pragma unroll
          for (int a = 0; a < NC; a++) b[r][a] = in.val(j, r, a);
        }
      if (j > 0) {
        // Schur complement of the previous block: K -= Kjm C^-1 Kjm^T, b -= Kjm C^-1 y, Kjm = K_{j,j-1} masked
        double Z[H][H];  // Z[:, r] = C^-1 Kjm[r, :]^T
#pragma unroll
        for (int r = 0; r < H; r++) {
          double z[H];
#pragma unroll
          for (int c = 0; c < H; c++) z[c] = ((fm >> r) & 1) || ((fmp >> c) & 1) ? 0.0 : sep[c][r];
          chol_solve<H>(Lp, z);
#pragma unroll
          for (int c = 0; c < H; c++) Z[c][r] = z[c];
        }
#pragma unroll
        for (int r = 0; r < H; r++) {
          if ((fm >> r) & 1) continue;
#pragma unroll
          for (int s = 0; s < H; s++) {
            double acc = 0.0;
#pragma unroll
            for (int c = 0; c < H; c++) acc += (((fmp >> c) & 1) ? 0.0 : sep[c][r]) * Z[c][s];
            K[r][s] -= acc;
          }
#pragma unroll
          for (int a = 0; a < NC; a++) {
            double acc = 0.0;
#pragma unroll
            for (int c = 0; c < H; c++) acc += Z[c][r] * yp[c][a];
            b[r][a] -= acc;
          }
        }
      }
      double L[6] = {0, 0, 0, 0, 0, 0};
      chol<H>(K, L);
#pragma unroll
      for (int q = 0; q < 6; q++) fac[(size_t)j * 6 + q] = Lp[q] = L[q];
#pragma unroll
      for (int r = 0; r < H; r++)
#pragma unroll
        for (int a = 0; a < NC; a++) D[(size_t)j * HN + r * NC + a] = yp[r][a] = b[r][a];
#pragma unroll
      for (int r = 0; r < H; r++)
#pragma unroll
        for (int c = 0; c < H; c++) { sep[r][c] = se[r][c]; eep[r][c] = ee[r][c]; }
      fmp = fm;
    }
    // back substitution: x_j = C_j^-1 (y_j - K_{j,j+1} x_{j+1}), K_{j,j+1} masked
    double xn[H][NC];
    int fmn = 0;
    for (int j = W - 1; j >= 0; j--) {
      const int fm = in.flags(j, H);
      double Lj[6];
#pragma unroll
      for (int q = 0; q < 6; q++) Lj[q] = fac[(size_t)j * 6 + q];
      double rhs[H][NC];
#pragma unroll
      for (int r = 0; r < H; r++)
#pragma unroll
        for (int a = 0; a < NC; a++) rhs[r][a] = D[(size_t)j * HN + r * NC + a];
      if (j < W - 1) {
        double ss[H][H], se[H][H], ee[H][H];
        seg_blocks<H>(seg_t[j], ss, se, ee);
#pragma unroll
        for (int r = 0; r < H; r++) {
          if ((fm >> r) & 1) continue;
#pragma unroll
          for (int c = 0; c < H; c++) {
            if ((fmn >> c) & 1) continue;
#pragma unroll
            for (int a = 0; a < NC; a++) rhs[r][a] -= se[r][c] * xn[c][a];
          }
        }
      }
#pragma unroll
      for (int a = 0; a < NC; a++) {
        double x[H];
#pragma unroll
        for (int r = 0; r < H; r++) x[r] = rhs[r][a];
        chol_solve<H>(Lj, x);
#pragma unroll
        for (int r = 0; r < H; r++) xn[r][a] = x[r];
      }
#pragma unroll
      for (int r = 0; r < H; r++)
#pragma unroll
        for (int a = 0; a < NC; a++) D[(size_t)j * HN + r * NC + a] = xn[r][a];
      fmn = fm;
    }
  }
  // fixed derivatives are the given values exactly; with two waypoints the free ones are 0
  for (int j = 0; j < W; j++) {
    const int fm = in.flags(j, H);
#pragma unroll
    for (int r = 0; r < H; r++)
#pragma unroll
      for (int a = 0; a < NC; a++)
        if ((fm >> r) & 1) D[(size_t)j * HN + r * NC + a] = in.val(j, r, a);
        else if (W == 2) D[(size_t)j * HN + r * NC + a] = 0.0;
  }
}

struct TrajArgs {
  int n_paths;
  const long long *offset;
  const mplx_waypoint *wps;
  const uint8_t *ctl;
  const double *dts;
  double v;
  int control, yaw_control, n_samples;
  int32_t *status;
  uint8_t *mono;  // per path: the running sum of segment times never decreases
  double *seg_t, *taus, *coeff, *samples;
  double *fac, *dpos, *dyaw;  // scratch: [n_wp*6], [n_wp*H*DIM], [n_wp*HY]
};

template <int DIM, int H, int HY>
__global__ void __launch_bounds__(128) traj_sweep_kernel(TrajArgs A) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A.n_paths) return;
  const long long b = A.offset[p];
  const int W = (int)(A.offset[p + 1] - b);
  const mplx_waypoint *w = A.wps + b;
  double *seg_t = A.seg_t + b, *taus = A.taus + b;
  // segment times (given, or TrajSolver::allocate_time: |p_j+1 - p_j|_inf / v) and their running sum, as
  // Trajectory's constructor adds them (trajectory.h:48-54)
  bool mono = true;
  if (W > 0) taus[0] = 0.0;
  for (int j = 0; j + 1 < W; j++) {
    double t;
    if (A.dts) {
      t = A.dts[b + j];
    } else {
      double d = 0.0;
#pragma unroll
      for (int a = 0; a < DIM; a++) {
        const double x = fabs(w[j + 1].pos[a] - w[j].pos[a]);
        if (x > d) d = x;
      }
      t = d / A.v;
    }
    seg_t[j] = t;
    taus[j + 1] = t + taus[j];
    mono = mono && taus[j + 1] >= taus[j];
  }
  if (W > 0) seg_t[W - 1] = 0.0;
  A.status[p] = W >= 2 ? 1 : 0;
  A.mono[p] = mono ? 1 : 0;
  if (W < 2) return;
  const uint8_t *ctl = A.ctl ? A.ctl + b : nullptr;
  const PathIn pin{w, ctl, A.control, W, false};
  sweep<H, DIM>(pin, seg_t, A.fac + b * 6, A.dpos + b * H * DIM);
  const PathIn yin{w, ctl, A.yaw_control, W, true};
  sweep<HY, 1>(yin, seg_t, A.fac + b * 6, A.dyaw + b * HY);
}

__device__ __forceinline__ int path_of(const long long *offset, int n_paths, long long slot) {
  int lo = 0, hi = n_paths - 1;  // the last path p with offset[p] <= slot
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (offset[mid] <= slot) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// every coefficient of one segment (axes, then yaw) is finite
template <int DIM>
__device__ __forceinline__ bool coeff_finite(const double *c) {
  bool finite = true;
  for (int k = 0; k < (DIM + 1) * 6; k++) finite = finite && isfinite(c[k]);
  return finite;
}

// Coefficients of one axis of one segment from the derivatives d0 (start) and d1 (end), as Primitive1D holds them
// (c[5-k] = k! p_k, p_k the coefficient of t^k).
template <int H>
__device__ __forceinline__ void seg_coeff(double tau, const double (&d0)[H], const double (&d1)[H], double *c) {
#pragma unroll
  for (int k = 0; k < 6; k++) c[k] = 0.0;
  double tp[2 * H];
  tp[0] = 1.0;
#pragma unroll
  for (int k = 1; k < 2 * H; k++) tp[k] = tp[k - 1] * tau;
  double t[H];  // tau^k (d1_k - sum_{n=k}^{h-1} d0_n tau^(n-k) / (n-k)!)
#pragma unroll
  for (int k = 0; k < H; k++) {
    double r = d1[k];
    double f = 1.0;
#pragma unroll
    for (int n = k; n < H; n++) {
      if (n > k) f *= (double)(n - k);
      r -= d0[n] * tp[n - k] / f;
    }
    t[k] = tp[k] * r;
  }
  double fact = 1.0;
#pragma unroll
  for (int k = 0; k < 2 * H; k++) {
    if (k > 0) fact *= (double)k;
    if (k < H) {
      c[5 - k] = d0[k];
    } else {
      double q = 0.0;
#pragma unroll
      for (int m = 0; m < H; m++) q += binv<H>(k - H, m) * t[m];
      c[5 - k] = q / tp[k] * fact;
    }
  }
}

template <int DIM, int H, int HY>
__global__ void __launch_bounds__(128) traj_coeff_kernel(TrajArgs A, long long n_wp) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < n_wp; s += (long long)gridDim.x * blockDim.x) {
    const int p = path_of(A.offset, A.n_paths, s);
    const long long b = A.offset[p];
    const int W = (int)(A.offset[p + 1] - b), j = (int)(s - b);
    double *c = A.coeff + s * (DIM + 1) * 6;
    if (j + 1 >= W) {  // the last slot of a path has no segment
      for (int k = 0; k < (DIM + 1) * 6; k++) c[k] = 0.0;
      continue;
    }
    const double tau = A.seg_t[s];
#pragma unroll
    for (int a = 0; a < DIM; a++) {
      double d0[H], d1[H];
#pragma unroll
      for (int k = 0; k < H; k++) {
        d0[k] = A.dpos[s * H * DIM + k * DIM + a];
        d1[k] = A.dpos[(s + 1) * H * DIM + k * DIM + a];
      }
      seg_coeff<H>(tau, d0, d1, c + a * 6);
    }
    {
      double d0[HY], d1[HY];
#pragma unroll
      for (int k = 0; k < HY; k++) {
        d0[k] = A.dyaw[s * HY + k];
        d1[k] = A.dyaw[(s + 1) * HY + k];
      }
      seg_coeff<HY>(tau, d0, d1, c + DIM * 6);
    }
    if (!coeff_finite<DIM>(c)) A.status[p] = 0;
  }
}

// include/mpl_basis/math.h power and Primitive1D's evaluators, in the host's operand order
__device__ __forceinline__ double power(double t, int n) {
  double tn = 1;
  while (n > 0) { tn *= t; n--; }
  return tn;
}
__device__ __forceinline__ double pr_p(const double *c, double t) {
  return c[0] / 120 * power(t, 5) + c[1] / 24 * power(t, 4) + c[2] / 6 * power(t, 3) + c[3] / 2 * t * t + c[4] * t + c[5];
}
__device__ __forceinline__ double pr_v(const double *c, double t) {
  return c[0] / 24 * power(t, 4) + c[1] / 6 * power(t, 3) + c[2] / 2 * t * t + c[3] * t + c[4];
}
__device__ __forceinline__ double pr_a(const double *c, double t) { return c[0] / 6 * power(t, 3) + c[1] / 2 * t * t + c[2] * t + c[3]; }
__device__ __forceinline__ double pr_j(const double *c, double t) { return c[0] / 2 * t * t + c[1] * t + c[2]; }

// One row of Trajectory::sample at polynomial time tau (already clamped) and real time `time`:
// Trajectory::evaluate(t, Command&) (trajectory.h:100-137) after its getTau and lambda lookup, in the host's
// operand order.  taus is the path's running sum of segment times (S + 1 entries), coeff its first segment's
// coefficients; mono says the running sum never decreases.  Leaves row untouched when no segment holds tau.
template <int DIM>
__device__ __forceinline__ void eval_row(const double *taus, int S, bool mono, const double *coeff, double tau,
                                         double time, double lambda, double lambda_dot, double *row) {
  // the first segment with taus[id] <= tau <= taus[id+1]; when the running sum never decreases, the first id
  // with taus[id+1] >= tau
  int id = -1;
  if (mono) {
    int lo = 0, hi = S - 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (taus[mid + 1] >= tau) hi = mid;
      else lo = mid + 1;
    }
    if (tau >= taus[lo] && tau <= taus[lo + 1]) id = lo;
  } else {
    for (int k = 0; k < S; k++)
      if (tau >= taus[k] && tau <= taus[k + 1]) { id = k; break; }
  }
  if (id < 0) return;
  tau -= taus[id];
  const double *c = coeff + (size_t)id * (DIM + 1) * 6;
  const double yaw = normalize_angle(pr_p(c + DIM * 6, tau));
  const double yaw_dot = normalize_angle(pr_v(c + DIM * 6, tau));
#pragma unroll
  for (int a = 0; a < DIM; a++) {
    const double *ca = c + a * 6;
    const double vel = pr_v(ca, tau) / lambda;
    const double acc = pr_a(ca, tau) / lambda / lambda - vel * lambda_dot / lambda / lambda / lambda;
    row[a] = pr_p(ca, tau);
    row[DIM + a] = vel;
    row[2 * DIM + a] = acc;
    row[3 * DIM + a] = pr_j(ca, tau) / lambda / lambda - 3 / power(lambda, 3) * acc * acc * lambda_dot +
                       3 / power(lambda, 4) * vel * lambda_dot * lambda_dot;
  }
  row[4 * DIM] = yaw;
  row[4 * DIM + 1] = yaw_dot;
  row[4 * DIM + 2] = time;
}

template <int DIM>
__global__ void __launch_bounds__(128) traj_sample_kernel(TrajArgs A) {
  const int per = A.n_samples + 1;
  constexpr int RW = 4 * DIM + 3;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < (long long)A.n_paths * per;
       g += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(g / per), i = (int)(g % per);
    double *o = A.samples + g * RW;
    double row[RW];
#pragma unroll
    for (int k = 0; k < RW; k++) row[k] = 0.0;
    if (A.status[p]) {
      const long long b = A.offset[p];
      const int S = (int)(A.offset[p + 1] - b) - 1;
      const double *taus = A.taus + b;
      const double total = taus[S];
      const double dt = total / A.n_samples;
      const double time = i * dt;
      double tau = time;
      if (tau < 0) tau = 0;
      if (tau > total) tau = total;
      eval_row<DIM>(taus, S, A.mono[p] != 0, A.coeff + b * (DIM + 1) * 6, tau, time, 1.0, 0.0, row);
    }
#pragma unroll
    for (int k = 0; k < RW; k++) o[k] = row[k];
  }
}

int order_of(int control) {  // h = N/2 of TrajSolver's PolySolver for this control, 0 when it has none
  switch (control) {
    case MPLX_VEL: case MPLX_VELxYAW: return 1;
    case MPLX_ACC: case MPLX_ACCxYAW: return 2;
    case MPLX_JRK: case MPLX_JRKxYAW: return 3;
    default: return 0;
  }
}

// control and yaw_control are VEL, ACC or JRK orders (mplx_traj_solve refuses SNP before any launch)
cudaError_t launch_solve(int dim, int control, int yaw_control, const TrajArgs &A, long long n_wp, cudaStream_t st,
                         int *launches) {
  return with_dim(dim, [&](auto DIM) {
    return with_order(control, [&](auto H) {
      return with_order(yaw_control, [&](auto HY) {
        if constexpr (H == 4 || HY == 4) {
          return cudaErrorInvalidValue;
        } else {
          if (cudaError_t e = launch(traj_sweep_kernel<DIM, H, HY>, A.n_paths, false, st, launches, A)) return e;
          if (n_wp > 0)
            if (cudaError_t e = launch(traj_coeff_kernel<DIM, H, HY>, n_wp, true, st, launches, A, n_wp)) return e;
          if (!A.samples) return cudaSuccess;
          return launch(traj_sample_kernel<DIM>, (long long)A.n_paths * (A.n_samples + 1), true, st, launches, A);
        }
      });
    });
  });
}

}  // namespace
}  // namespace mplx

extern "C" int mplx_traj_solve(mplx_ctx *c, int n_paths, const int64_t *offset, const mplx_waypoint *wps,
                               const uint8_t *wp_control, const double *dts, double v, int control, int yaw_control,
                               int n_samples, mplx_traj_out *out) {
  if (int r = mplx_bind(c)) return r;
  const int h = mplx::order_of(control);
  if (h == 0) return fail(MPLX_ERR_ARG, "control 0x%x: TrajSolver solves VEL, ACC and JRK (with or without YAW)", control);
  const int hy = (yaw_control == MPLX_VEL || yaw_control == MPLX_ACC || yaw_control == MPLX_JRK) ? mplx::order_of(yaw_control) : 0;
  if (hy == 0) return fail(MPLX_ERR_ARG, "yaw_control 0x%x: must be VEL, ACC or JRK", yaw_control);
  if (!dts && !(v > 0)) return fail(MPLX_ERR_ARG, "no segment times: dts is NULL and v <= 0");
  long long n_wp = 0;
  if (int r = mplx::check_batch(n_paths, offset, out && out->status && out->seg_t && out->coeff, wps != nullptr,
                                out && out->samples, n_samples, n_wp))
    return r;
  out->seconds = 0.0;
  if (n_paths == 0) return MPLX_OK;
  const int dim = c->dim;
  TrajBufs &B = c->tb;
  const size_t nw = (size_t)std::max<long long>(n_wp, 1);
  CU(B.offset.reserve(n_paths + 1)); CU(B.status.reserve(n_paths)); CU(B.mono.reserve(n_paths));
  CU(B.wps.reserve(nw)); CU(B.seg_t.reserve(nw)); CU(B.taus.reserve(nw));
  CU(B.coeff.reserve(nw * (dim + 1) * 6)); CU(B.fac.reserve(nw * 6)); CU(B.dpos.reserve(nw * h * dim));
  CU(B.dyaw.reserve(nw * hy));
  if (wp_control) CU(B.ctl.reserve(nw));
  if (dts) CU(B.dts.reserve(nw));
  const size_t n_rows = out->samples ? (size_t)n_paths * (n_samples + 1) : 0;
  if (out->samples) CU(B.samples.reserve(n_rows * (4 * dim + 3)));
  cudaStream_t st = c->stream;
  static_assert(sizeof(long long) == sizeof(int64_t), "offset width");
  CU(cudaMemcpyAsync(B.offset.p, offset, sizeof(int64_t) * (n_paths + 1), cudaMemcpyHostToDevice, st));
  if (n_wp > 0) {
    CU(cudaMemcpyAsync(B.wps.p, wps, sizeof(mplx_waypoint) * n_wp, cudaMemcpyHostToDevice, st));
    if (wp_control) CU(cudaMemcpyAsync(B.ctl.p, wp_control, (size_t)n_wp, cudaMemcpyHostToDevice, st));
    if (dts) CU(cudaMemcpyAsync(B.dts.p, dts, sizeof(double) * n_wp, cudaMemcpyHostToDevice, st));
  }
  mplx::TrajArgs A{n_paths, B.offset.p, B.wps.p, wp_control ? B.ctl.p : nullptr, dts ? B.dts.p : nullptr, v, control,
                   yaw_control, n_samples, B.status.p, B.mono.p, B.seg_t.p, B.taus.p, B.coeff.p,
                   out->samples ? B.samples.p : nullptr, B.fac.p, B.dpos.p, B.dyaw.p};
  TimedRun timed;
  CU(timed.run(st, c->launches,
               [&](int *launches) { return mplx::launch_solve(dim, control, yaw_control, A, n_wp, st, launches); }));
  CU(cudaMemcpyAsync(out->status, B.status.p, sizeof(int32_t) * n_paths, cudaMemcpyDeviceToHost, st));
  if (n_wp > 0) {
    CU(cudaMemcpyAsync(out->seg_t, B.seg_t.p, sizeof(double) * n_wp, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out->coeff, B.coeff.p, sizeof(double) * n_wp * (dim + 1) * 6, cudaMemcpyDeviceToHost, st));
  }
  if (out->samples) CU(cudaMemcpyAsync(out->samples, B.samples.p, sizeof(double) * n_rows * (4 * dim + 3), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(timed.seconds(&out->seconds));
  return MPLX_OK;
}

// ---- time scaling of trajectories (mplx_traj_scale, include/mplx.h) -------------------------------------------
//   scale_prep_kernel    one thread per path: parameter and duration checks, the running sum of segment times
//   scale_cand_kernel    one thread per segment: finite coefficients; for SCALE_DOWN the knots of the segment's
//                        axes (max_vel, extrema_v), sorted by time
//   scale_knot_kernel    one thread per path: max_l, the knot list with equal times merged
//   scale_fit_kernel     one thread per lambda slot: the LambdaSeg fit of knots k and k + 1
//   scale_times_kernel   one thread per path: the running sum of dT, the scaled waypoint times Ts
//   scale_sample_kernel  one thread per sample: getTau, the lambda lookup and eval_row
// Within a path the knots of segment j lie in [taus[j], taus[j+1]] (a root tv in (0, t) rounds to
// tv + taus[j] <= t + taus[j]), so sorting each segment's knots and concatenating them in segment order sorts
// the path's knots as std::sort does, up to the order of equal times, which the merge makes irrelevant
// (DESIGN.md §8).
namespace mplx {
namespace {

constexpr int kCand = 5;  // knots per segment and axis: <= 3 extrema_v roots, the start and the end

// math.h:21-131 (quad, cubic, quartic, solve), operation by operation; r receives the roots in the host's order
__device__ __forceinline__ int quad_roots(double b, double c, double d, double *r) {
  const double p = c * c - 4 * b * d;
  if (p < 0) return 0;
  r[0] = (-c - sqrt(p)) / (2 * b);
  r[1] = (-c + sqrt(p)) / (2 * b);
  return 2;
}
__device__ __forceinline__ int cubic_roots(double a, double b, double c, double d, double *r) {
  const double a2 = b / a, a1 = c / a, a0 = d / a;
  const double Q = (3 * a1 - a2 * a2) / 9;
  const double R = (9 * a1 * a2 - 27 * a0 - 2 * a2 * a2 * a2) / 54;
  const double D = Q * Q * Q + R * R;
  if (D > 0) {
    const double S = cbrt(R + sqrt(D));
    const double T = cbrt(R - sqrt(D));
    r[0] = -a2 / 3 + (S + T);
    return 1;
  }
  if (D == 0) {
    const double S = cbrt(R);
    r[0] = -a2 / 3 + S + S;
    r[1] = -a2 / 3 - S;
    return 2;
  }
  const double theta = acos(R / sqrt(-Q * Q * Q));
  r[0] = 2 * sqrt(-Q) * cos(theta / 3) - a2 / 3;
  r[1] = 2 * sqrt(-Q) * cos((theta + 2 * MPLX_PI) / 3) - a2 / 3;
  r[2] = 2 * sqrt(-Q) * cos((theta + 4 * MPLX_PI) / 3) - a2 / 3;
  return 3;
}
__device__ __forceinline__ int quartic_roots(double a, double b, double c, double d, double e, double *r) {
  const double a3 = b / a, a2 = c / a, a1 = d / a, a0 = e / a;
  double ys[3];
  cubic_roots(1, -a2, a1 * a3 - 4 * a0, 4 * a2 * a0 - a1 * a1 - a3 * a3 * a0, ys);
  const double y1 = ys[0];
  const double rr = a3 * a3 / 4 - a2 + y1;
  if (rr < 0) return 0;
  const double R = sqrt(rr);
  double D, E;
  if (R != 0) {
    D = sqrt(0.75 * a3 * a3 - R * R - 2 * a2 + 0.25 * (4 * a3 * a2 - 8 * a1 - a3 * a3 * a3) / R);
    E = sqrt(0.75 * a3 * a3 - R * R - 2 * a2 - 0.25 * (4 * a3 * a2 - 8 * a1 - a3 * a3 * a3) / R);
  } else {
    D = sqrt(0.75 * a3 * a3 - 2 * a2 + 2 * sqrt(y1 * y1 - 4 * a0));
    E = sqrt(0.75 * a3 * a3 - 2 * a2 - 2 * sqrt(y1 * y1 - 4 * a0));
  }
  int n = 0;
  if (!isnan(D)) {
    r[n++] = -a3 / 4 + R / 2 + D / 2;
    r[n++] = -a3 / 4 + R / 2 - D / 2;
  }
  if (!isnan(E)) {
    r[n++] = -a3 / 4 - R / 2 + E / 2;
    r[n++] = -a3 / 4 - R / 2 - E / 2;
  }
  return n;
}
__device__ __forceinline__ int solve_roots(double a, double b, double c, double d, double e, double *r) {
  if (a != 0) return quartic_roots(a, b, c, d, e, r);
  if (b != 0) return cubic_roots(b, c, d, e, r);
  if (c != 0) return quad_roots(c, d, e, r);
  if (d != 0) { r[0] = -e / d; return 1; }
  return 0;
}

// Primitive1D::extrema_v (primitive.h:152-162): roots of a(t) in (0, t), stopping at the first root >= t
__device__ __forceinline__ int extrema_v(const double *c, double t, double *ts) {
  double r[4];
  const int n = solve_roots(0, c[0] / 6, c[1] / 2, c[2], c[3], r);
  int m = 0;
  for (int k = 0; k < n; k++) {
    if (r[k] > 0 && r[k] < t) ts[m++] = r[k];
    else if (r[k] >= t) break;
  }
  return m;
}
// Primitive::max_vel (primitive.h:353-363)
__device__ __forceinline__ double max_vel(const double *c, double t) {
  double ts[3];
  const int n = extrema_v(c, t, ts);
  const double v0 = fabs(pr_v(c, 0)), v1 = fabs(pr_v(c, t));
  double m = v0 < v1 ? v1 : v0;  // std::max
  for (int k = 0; k < n; k++)
    if (ts[k] > 0 && ts[k] < t) {
      const double v = fabs(pr_v(c, ts[k]));
      m = v > m ? v : m;
    }
  return m;
}

// Primitive1D::extrema_a (primitive.h:169-179) with Primitive::max_acc (:369-379)
__device__ __forceinline__ double max_acc(const double *c, double t) {
  double r[4];
  const int n = solve_roots(0, 0, c[0] / 2, c[1], c[2], r);
  const double a0 = fabs(pr_a(c, 0)), a1 = fabs(pr_a(c, t));
  double m = a0 < a1 ? a1 : a0;  // std::max
  for (int k = 0; k < n; k++) {
    if (r[k] > 0 && r[k] < t) {
      const double a = fabs(pr_a(c, r[k]));
      m = a > m ? a : m;
    } else if (r[k] >= t) {
      break;
    }
  }
  return m;
}
// Primitive1D::extrema_j (primitive.h:186-193) with Primitive::max_jrk (:384-394)
__device__ __forceinline__ double max_jrk(const double *c, double t) {
  const double j0 = fabs(pr_j(c, 0)), j1 = fabs(pr_j(c, t));
  double m = j0 < j1 ? j1 : j0;
  if (c[0] != 0) {
    const double ts = -c[1] * 2 / c[0];
    if (ts > 0 && ts < t) {
      const double j = fabs(pr_j(c, ts));
      m = j > m ? j : m;
    }
  }
  return m;
}

// LambdaSeg (lambda.h:24-71): the Hermite fit by Gauss-Jordan inversion as on the host (mpl_host.hpp)
struct LSeg {
  double a[4], ti, tf, dT;
};
__device__ __forceinline__ double lseg_T(const double *a, double t) {
  return a[0] / 4 * power(t, 4) + a[1] / 3 * power(t, 3) + a[2] / 2 * t * t + a[3] * t;
}
__device__ void lseg_fit(double t1, double p1, double t2, double p2, LSeg &s) {
  double A[4][4] = {{power(t1, 3), t1 * t1, t1, 1}, {3 * t1 * t1, 2 * t1, 1, 0},
                    {power(t2, 3), t2 * t2, t2, 1}, {3 * t2 * t2, 2 * t2, 1, 0}};
  double inv[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
#pragma unroll
  for (int col = 0; col < 4; col++) {
    int piv = col;
#pragma unroll
    for (int r = col + 1; r < 4; r++)
      if (fabs(A[r][col]) > fabs(A[piv][col])) piv = r;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      // a row exchange without dynamic register indexing
      double x = A[col][k], y = inv[col][k];
#pragma unroll
      for (int r = col + 1; r < 4; r++)
        if (r == piv) {
          A[col][k] = A[r][k]; A[r][k] = x;
          inv[col][k] = inv[r][k]; inv[r][k] = y;
        }
    }
    const double d = A[col][col];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      A[col][k] /= d;
      inv[col][k] /= d;
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
      if (r == col) continue;
      const double f = A[r][col];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        A[r][k] -= f * A[col][k];
        inv[r][k] -= f * inv[col][k];
      }
    }
  }
  const double b[4] = {p1, 0.0, p2, 0.0};
#pragma unroll
  for (int i = 0; i < 4; i++) {
    double acc = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) acc += inv[i][k] * b[k];
    s.a[i] = fabs(acc) < 1e-5 ? 0.0 : acc;
  }
  s.ti = t1;
  s.tf = t2;
  s.dT = lseg_T(s.a, t2) - lseg_T(s.a, t1);
}

struct ScaleArgs {
  int n_paths, mode, n_samples;
  const long long *offset;
  const double *seg_t, *coeff, *par;  // par: [3 * n_paths] mv, ri, rf
  int32_t *status, *n_cand, *n_knot;
  double *taus, *cand, *cand_p, *knot_t, *knot_p, *lam, *lam_T, *total, *seg_T, *samples;
  uint8_t *lam_mono;
};

__device__ __forceinline__ bool pos_finite(double x) { return isfinite(x) && x > 0; }

// Trajectory's constructor for the path of W waypoints at slot b: taus[j+1] = t_j + taus[j].  Returns ok and
// whether every segment time t_j is positive and finite.
__device__ __forceinline__ bool seg_taus(const double *seg_t, double *taus, long long b, int W, bool ok) {
  if (W > 0) taus[b] = 0.0;
  for (int j = 0; j + 1 < W; j++) {
    const double t = seg_t[b + j];
    ok = ok && pos_finite(t);
    taus[b + j + 1] = t + taus[b + j];
  }
  return ok;
}

// Lambda::getTau's running T += dT over nl lambda segments, left to right, into lT[0, nl].  Returns whether it
// never decreases.
__device__ __forceinline__ bool lam_sums(const double *lam, int nl, double *lT) {
  double T = 0;
  bool mono = true;
  lT[0] = 0;
  for (int k = 0; k < nl; k++) {
    const double Tn = T + lam[k * 7 + 6];
    mono = mono && Tn >= T;
    lT[k + 1] = T = Tn;
  }
  return mono;
}

template <int DIM>
__global__ void __launch_bounds__(128) scale_prep_kernel(ScaleArgs A) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A.n_paths) return;
  const long long b = A.offset[p];
  const int W = (int)(A.offset[p + 1] - b);
  const double *par = A.par + 3 * p;
  const bool ok = W >= 2 && pos_finite(par[1]) && pos_finite(par[2]) && (A.mode == MPLX_TRAJ_SCALE || pos_finite(par[0]));
  A.status[p] = seg_taus(A.seg_t, A.taus, b, W, ok) ? 1 : 0;
}

template <int DIM>
__global__ void __launch_bounds__(128) scale_cand_kernel(ScaleArgs A, long long n_wp) {
  constexpr int NC = kCand * DIM;
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < n_wp; s += (long long)gridDim.x * blockDim.x) {
    const int p = path_of(A.offset, A.n_paths, s);
    const long long b = A.offset[p];
    const int W = (int)(A.offset[p + 1] - b), j = (int)(s - b);
    A.n_cand[s] = 0;
    if (j + 1 >= W) continue;
    const double *c = A.coeff + s * (DIM + 1) * 6;
    const bool finite = coeff_finite<DIM>(c);
    if (!finite) A.status[p] = 0;  // every writer stores 0
    if (A.mode != MPLX_TRAJ_SCALE_DOWN || !finite) continue;
    const double t = A.seg_t[s], mv = A.par[3 * p], tau0 = A.taus[s];
    double kt[NC], pmax = 0.0;
    int n = 0;
    for (int i = 0; i < DIM; i++) {
      const double *ci = c + i * 6;
      if (!(max_vel(ci, t) > mv)) continue;
      double ts[kCand];
      int m = extrema_v(ci, t, ts);
      if (j != 0) ts[m++] = 0;
      ts[m++] = t;
      for (int k = 0; k < m; k++) {
        const double lv = fabs(pr_v(ci, ts[k])) / mv;
        if (lv <= 1) continue;
        // insertion by time
        const double tk = ts[k] + tau0;
        int q = n++;
        while (q > 0 && kt[q - 1] > tk) { kt[q] = kt[q - 1]; q--; }
        kt[q] = tk;
        pmax = lv > pmax ? lv : pmax;
      }
    }
    for (int k = 0; k < n; k++) A.cand[s * NC + k] = kt[k];
    A.n_cand[s] = n;
    A.cand_p[s] = pmax;
  }
}

// Trajectory::scale_down's knot list (trajectory.h:173-228 as the host defines it), or scale's two knots
template <int DIM>
__global__ void __launch_bounds__(128) scale_knot_kernel(ScaleArgs A) {
  constexpr int NC = kCand * DIM;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A.n_paths) return;
  const long long b = A.offset[p];
  const int S = (int)(A.offset[p + 1] - b) - 1;
  double *kt = A.knot_t + b * NC, *kp = A.knot_p + b * NC;
  A.n_knot[p] = 0;
  if (!A.status[p]) return;
  const double *par = A.par + 3 * p;
  const double T = A.taus[b + S];
  if (A.mode == MPLX_TRAJ_SCALE) {
    kt[0] = 0; kp[0] = 1.0 / par[1];
    kt[1] = T; kp[1] = 1.0 / par[2];
    A.n_knot[p] = 2;
    return;
  }
  const double ri = par[1], rf = par[2];
  double max_l = 1;
  if (ri > max_l) max_l = ri;
  for (int j = 0; j < S; j++)
    if (A.n_cand[b + j] && A.cand_p[b + j] > max_l) max_l = A.cand_p[b + j];
  if (rf > max_l) max_l = rf;
  if (max_l <= 1) {
    A.status[p] = 2;
    return;
  }
  // the sorted knots with equal times merged into their first: (0, ri), every interior time with max_l, and
  // (T, rf) unless a knot of the last segment ends there too, which then comes first and keeps max_l
  int n = 1;
  kt[0] = 0; kp[0] = ri;
  for (int j = 0; j < S; j++) {
    const int m = A.n_cand[b + j];
    const double *ct = A.cand + (b + j) * NC;
    for (int k = 0; k < m; k++)
      if (ct[k] > kt[n - 1]) { kt[n] = ct[k]; kp[n] = max_l; n++; }
  }
  if (T > kt[n - 1]) { kt[n] = T; kp[n] = rf; n++; }
  A.n_knot[p] = n;
}

template <int DIM>
__global__ void __launch_bounds__(128) scale_fit_kernel(ScaleArgs A, long long n_slot) {
  constexpr int NC = kCand * DIM;
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < n_slot; s += (long long)gridDim.x * blockDim.x) {
    const int p = path_of(A.offset, A.n_paths, s / NC);
    const long long b = A.offset[p] * NC;
    const int k = (int)(s - b);
    double *o = A.lam + s * 7;
    LSeg g = {{0, 0, 0, 0}, 0, 0, 0};
    if (k + 1 < A.n_knot[p]) lseg_fit(A.knot_t[s], A.knot_p[s], A.knot_t[s + 1], A.knot_p[s + 1], g);
    o[0] = g.a[0]; o[1] = g.a[1]; o[2] = g.a[2]; o[3] = g.a[3]; o[4] = g.ti; o[5] = g.tf; o[6] = g.dT;
  }
}

template <int DIM>
__global__ void __launch_bounds__(128) scale_times_kernel(ScaleArgs A) {
  constexpr int NC = kCand * DIM;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A.n_paths) return;
  const long long b = A.offset[p];
  const int W = (int)(A.offset[p + 1] - b), S = W - 1;
  double *segT = A.seg_T + b;
  const double *taus = A.taus + b;
  const int st = A.status[p];
  if (st == 0) {
    for (int j = 0; j < W; j++) segT[j] = 0.0;
    A.total[p] = 0.0;
    return;
  }
  if (st == 2) {  // no lambda: Ts = taus
    for (int j = 0; j < S; j++) segT[j] = taus[j + 1] - taus[j];
    segT[S] = 0.0;
    A.total[p] = taus[S];
    A.lam_mono[p] = 1;
    return;
  }
  const int nl = A.n_knot[p] - 1;
  const double *lam = A.lam + b * NC * 7;
  double *lT = A.lam_T + b * NC;
  A.lam_mono[p] = lam_sums(lam, nl, lT) ? 1 : 0;
  // Lambda::getT(taus[j]): the first segment with ti <= tau <= tf; the knots increase strictly from 0 and the
  // taus never decrease, so that segment's index never decreases along the path
  int k = 0;
  double prev = 0;
  for (int j = 0; j <= S; j++) {
    const double tau = taus[j];
    while (k < nl && !(tau >= lam[k * 7 + 4] && tau <= lam[k * 7 + 5])) k++;
    const double *a = lam + k * 7;
    const double Ts = k < nl ? lT[k] + (lseg_T(a, tau) - lseg_T(a, a[4])) : lT[nl];
    if (j > 0) segT[j - 1] = Ts - prev;
    prev = Ts;
  }
  segT[S] = 0.0;
  A.total[p] = prev;
}

// Lambda::getTau (lambda.h:157-179): -1 when no segment gives a root
__device__ __forceinline__ double get_tau(const double *lam, const double *lT, int nl, bool mono, double t) {
  int k = 0;
  if (mono) {  // skip the segments whose [T, T + dT] ends below t; the rest are scanned as on the host
    int lo = 0, hi = nl;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (lT[mid + 1] >= t) hi = mid;
      else lo = mid + 1;
    }
    k = lo;
  }
  for (; k < nl; k++) {
    if (t >= lT[k] && t <= lT[k + 1]) {
      const double *a = lam + k * 7;
      const double e = lT[k] - t - lseg_T(a, a[4]);
      double r[4];
      const int n = solve_roots(a[0] / 4, a[1] / 3, a[2] / 2, a[3], e, r);
      for (int q = 0; q < n; q++)
        if (r[q] >= a[4] && r[q] <= a[5]) return r[q];
    } else if (mono && t < lT[k]) {
      break;
    }
  }
  return -1;
}

// Trajectory::evaluate(time, Command&) (trajectory.h:100-137) of a path whose segment times are all positive:
// getTau, the clamp of tau to [0, total], the lambda lookup and eval_row.  nl = 0: no lambda (tau = time).
template <int DIM>
__device__ __forceinline__ void traj_row(const double *taus, int S, const double *coeff, const double *lam,
                                         const double *lT, int nl, bool lam_mono, double total, double time,
                                         double *row) {
  double tau = time, lambda = 1, lambda_dot = 0;
  if (nl > 0) tau = get_tau(lam, lT, nl, lam_mono, time);
  if (tau < 0) tau = 0;
  if (tau > total) tau = total;
  if (nl > 0) {
    // Lambda::evaluate: the first segment with ti <= tau < tf, else (tau at the last tf) the last one
    int lo = 0, hi = nl - 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (lam[mid * 7 + 5] > tau) hi = mid;
      else lo = mid + 1;
    }
    const double *a = lam + lo * 7;
    lambda = a[0] * power(tau, 3) + a[1] * tau * tau + a[2] * tau + a[3];
    lambda_dot = 3 * a[0] * tau * tau + 2 * a[1] * tau + a[2];
  }
  // the running sum of positive segment times never decreases
  eval_row<DIM>(taus, S, true, coeff, tau, time, lambda, lambda_dot, row);
}

template <int DIM>
__global__ void __launch_bounds__(128) scale_sample_kernel(ScaleArgs A) {
  constexpr int NC = kCand * DIM;
  const int per = A.n_samples + 1;
  constexpr int RW = 4 * DIM + 3;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < (long long)A.n_paths * per;
       g += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(g / per), i = (int)(g % per);
    double row[RW];
#pragma unroll
    for (int k = 0; k < RW; k++) row[k] = 0.0;
    const int st = A.status[p];
    if (st) {
      const long long b = A.offset[p];
      const int S = (int)(A.offset[p + 1] - b) - 1;
      const double total = A.total[p];
      const double dt = total / A.n_samples;
      const int nl = st == 1 ? A.n_knot[p] - 1 : 0;
      traj_row<DIM>(A.taus + b, S, A.coeff + b * (DIM + 1) * 6, A.lam + b * NC * 7, A.lam_T + b * NC, nl,
                    A.lam_mono[p] != 0, total, i * dt, row);
    }
    double *o = A.samples + g * RW;
#pragma unroll
    for (int k = 0; k < RW; k++) o[k] = row[k];
  }
}

cudaError_t launch_scale(int dim, const ScaleArgs &A, long long n_wp, cudaStream_t st, int *launches) {
  return with_dim(dim, [&](auto DIM) {
    const long long n_slot = n_wp * kCand * DIM;
    if (cudaError_t e = launch(scale_prep_kernel<DIM>, A.n_paths, false, st, launches, A)) return e;
    if (cudaError_t e = launch(scale_cand_kernel<DIM>, n_wp, true, st, launches, A, n_wp)) return e;
    if (cudaError_t e = launch(scale_knot_kernel<DIM>, A.n_paths, false, st, launches, A)) return e;
    if (cudaError_t e = launch(scale_fit_kernel<DIM>, n_slot, true, st, launches, A, n_slot)) return e;
    if (cudaError_t e = launch(scale_times_kernel<DIM>, A.n_paths, false, st, launches, A)) return e;
    if (!A.samples) return cudaSuccess;
    return launch(scale_sample_kernel<DIM>, (long long)A.n_paths * (A.n_samples + 1), true, st, launches, A);
  });
}

}  // namespace
}  // namespace mplx

extern "C" int mplx_traj_scale(mplx_ctx *c, int n_paths, const int64_t *offset, const double *seg_t,
                               const double *coeff, int mode, const double *mv, const double *ri, const double *rf,
                               int n_samples, mplx_traj_scale_out *out) {
  if (int r = mplx_bind(c)) return r;
  if (mode != MPLX_TRAJ_SCALE && mode != MPLX_TRAJ_SCALE_DOWN) return fail(MPLX_ERR_ARG, "mode %d: must be MPLX_TRAJ_SCALE or MPLX_TRAJ_SCALE_DOWN", mode);
  if (mode == MPLX_TRAJ_SCALE_DOWN && !mv) return fail(MPLX_ERR_ARG, "SCALE_DOWN without mv");
  long long n_wp = 0;
  if (int r = mplx::check_batch(n_paths, offset, ri && rf && out && out->status && out->total_t && out->seg_T,
                                seg_t && coeff, out && out->samples, n_samples, n_wp))
    return r;
  out->seconds = 0.0;
  if (n_paths == 0) return MPLX_OK;
  const int dim = c->dim;
  const size_t NC = (size_t)mplx::kCand * dim;
  TrajBufs &B = c->tb;
  const size_t nw = (size_t)std::max<long long>(n_wp, 1);
  CU(B.offset.reserve(n_paths + 1)); CU(B.status.reserve(n_paths)); CU(B.mono.reserve(n_paths));
  CU(B.par.reserve(3 * (size_t)n_paths)); CU(B.n_knot.reserve(n_paths)); CU(B.total.reserve(n_paths));
  CU(B.seg_t.reserve(nw)); CU(B.taus.reserve(nw)); CU(B.seg_T.reserve(nw)); CU(B.n_cand.reserve(nw));
  CU(B.cand_p.reserve(nw)); CU(B.coeff.reserve(nw * (dim + 1) * 6));
  CU(B.cand.reserve(nw * NC)); CU(B.knot_t.reserve(nw * NC)); CU(B.knot_p.reserve(nw * NC));
  CU(B.lam.reserve(nw * NC * 7)); CU(B.lam_T.reserve(nw * NC));
  const size_t n_rows = out->samples ? (size_t)n_paths * (n_samples + 1) : 0;
  if (out->samples) CU(B.samples.reserve(n_rows * (4 * dim + 3)));
  std::vector<double> par(3 * (size_t)n_paths);
  for (int p = 0; p < n_paths; p++) {
    par[3 * p] = mv ? mv[p] : 0.0;
    par[3 * p + 1] = ri[p];
    par[3 * p + 2] = rf[p];
  }
  cudaStream_t st = c->stream;
  CU(cudaMemcpyAsync(B.offset.p, offset, sizeof(int64_t) * (n_paths + 1), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(B.par.p, par.data(), sizeof(double) * par.size(), cudaMemcpyHostToDevice, st));
  if (n_wp > 0) {
    CU(cudaMemcpyAsync(B.seg_t.p, seg_t, sizeof(double) * n_wp, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(B.coeff.p, coeff, sizeof(double) * n_wp * (dim + 1) * 6, cudaMemcpyHostToDevice, st));
  }
  mplx::ScaleArgs A{n_paths, mode, n_samples, B.offset.p, B.seg_t.p, B.coeff.p, B.par.p, B.status.p, B.n_cand.p,
                    B.n_knot.p, B.taus.p, B.cand.p, B.cand_p.p, B.knot_t.p, B.knot_p.p, B.lam.p, B.lam_T.p,
                    B.total.p, B.seg_T.p, out->samples ? B.samples.p : nullptr, B.mono.p};
  TimedRun timed;
  CU(timed.run(st, c->launches, [&](int *launches) { return mplx::launch_scale(dim, A, n_wp, st, launches); }));
  CU(cudaMemcpyAsync(out->status, B.status.p, sizeof(int32_t) * n_paths, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(out->total_t, B.total.p, sizeof(double) * n_paths, cudaMemcpyDeviceToHost, st));
  if (n_wp > 0) CU(cudaMemcpyAsync(out->seg_T, B.seg_T.p, sizeof(double) * n_wp, cudaMemcpyDeviceToHost, st));
  std::vector<int32_t> nk;
  if (out->n_lambda) {
    nk.resize(n_paths);
    CU(cudaMemcpyAsync(nk.data(), B.n_knot.p, sizeof(int32_t) * n_paths, cudaMemcpyDeviceToHost, st));
  }
  if (out->lambda && n_wp > 0) CU(cudaMemcpyAsync(out->lambda, B.lam.p, sizeof(double) * n_wp * NC * 7, cudaMemcpyDeviceToHost, st));
  if (out->samples) CU(cudaMemcpyAsync(out->samples, B.samples.p, sizeof(double) * n_rows * (4 * dim + 3), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (out->n_lambda)
    for (int p = 0; p < n_paths; p++) out->n_lambda[p] = out->status[p] == 1 ? nk[p] - 1 : 0;
  CU(timed.seconds(&out->seconds));
  return MPLX_OK;
}

// ---- checking trajectories against the map and the limits (mplx_traj_check, include/mplx.h) -------------------
//   check_path_kernel    one thread per path: segment-time checks, the running sums of segment times and of the
//                        lambda segments' dT, the total time and N = ceil(v_max * total / res)
//   check_seg_kernel     one thread per segment: finite coefficients; is_free(segment) over its n + 1 samples
//                        and validate_primitive
//   check_sample_kernel  one warp per path: traverse_trajectory over the N + 1 samples, 32 at a time.  Lane l
//                        takes sample base + l; the previous sample's cell index comes from lane l - 1, and from
//                        the chunk before for lane 0.  The first counted sample that returns +inf ends the path
//                        (a ballot); with a potential map the chunk's terms are added to the running cost one
//                        lane after another in sample order, so the sum is the host's left-to-right sum.
namespace mplx {
namespace {

struct CheckArgs {
  int n_paths;
  const long long *offset;
  const double *seg_t, *coeff;
  const double *total_in, *lam;  // NULL: no path is scaled
  const int32_t *n_lam;
  const uint8_t *ctl;
  int32_t *status, *n_pts;  // n_pts: N of traverse_trajectory, 0 when outside [1, MPLX_SAMPLE_N_MAX]
  uint8_t *form;            // per path: at least 2 waypoints, every segment time and coefficient usable
  uint8_t *lam_mono;
  double *taus, *lam_T, *total, *cost;
  uint8_t *seg_free, *seg_valid;  // NULL: not asked for
};

template <int DIM>
__global__ void __launch_bounds__(128) check_path_kernel(const __grid_constant__ EnvParams P, CheckArgs A) {
  constexpr int NC = kCand * DIM;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A.n_paths) return;
  const long long b = A.offset[p];
  const int W = (int)(A.offset[p + 1] - b);
  const bool ok = seg_taus(A.seg_t, A.taus, b, W, W >= 2);
  // Lambda::getTau's running T += dT, as mplx_traj_scale keeps it
  const int nl = A.lam ? A.n_lam[p] : 0;
  bool mono = true;
  if (nl > 0) mono = lam_sums(A.lam + b * NC * 7, nl, A.lam_T + b * NC);
  A.lam_mono[p] = mono ? 1 : 0;
  const double total = nl > 0 ? A.total_in[p] : (W > 0 ? A.taus[b + W - 1] : 0.0);
  A.total[p] = total;
  const double nd = ceil(P.v_max * total / P.res);
  A.n_pts[p] = nd >= 1 && nd <= MPLX_SAMPLE_N_MAX ? (int)nd : 0;
  A.form[p] = ok ? 1 : 0;
}

// env_map::is_free(pr) (env_map.h:60-76) of one segment
template <int DIM>
__device__ bool seg_is_free(const EnvParams &P, const double *c, double t) {
  double max_v = 0;
#pragma unroll
  for (int a = 0; a < DIM; a++) {
    const double mv = max_vel(c + a * 6, t);
    if (mv > max_v) max_v = mv;
  }
  const double nd = ceil(max_v * t / P.res);
  if (!(nd <= MPLX_SAMPLE_N_MAX)) return false;
  const int n = (int)nd;
  const double dt = t / n;  // n = 0: every sample time is 0 * inf = NaN, outside the map
  for (int i = 0; i <= n; i++) {
    int pn[DIM];
    bool inside = true;
#pragma unroll
    for (int a = 0; a < DIM; a++) {
      pn[a] = float_to_int(pr_p(c + a * 6, i * dt), P.origin[a], P.res);
      inside = inside && (unsigned)pn[a] < (unsigned)P.mdim[a];
    }
    if (!inside) return false;
    int idx = pn[0] + P.mdim[0] * pn[1];
    if (DIM == 3) idx += P.mdim[0] * P.mdim[1] * pn[DIM - 1];
    if ((__ldg(P.occ_bits + (idx >> 5)) >> (idx & 31)) & 1u) return false;
    if (P.region_bits != nullptr && !((__ldg(P.region_bits + (idx >> 5)) >> (idx & 31)) & 1u)) return false;
  }
  return true;
}

// validate_xxx (primitive.h:476-493): ORD 1 max_vel, 2 max_acc, 3 max_jrk of every axis within mx
template <int DIM, int ORD>
__device__ bool validate_axes(const double *c, double t, double mx) {
  if (mx <= 0) return true;
  for (int a = 0; a < DIM; a++) {
    const double m = ORD == 1 ? max_vel(c + a * 6, t) : ORD == 2 ? max_acc(c + a * 6, t) : max_jrk(c + a * 6, t);
    if (m > mx) return false;
  }
  return true;
}

// validate_yaw (primitive.h:503-525): the velocity's direction against the yaw at both ends
template <int DIM>
__device__ bool validate_yaw_ends(const EnvParams &P, const double *c, double t) {
  if (P.yaw_max <= 0) return true;
  for (int e = 0; e < 2; e++) {
    const double te = e == 0 ? 0.0 : t;
    const double v0 = pr_v(c, te), v1 = pr_v(c + 6, te);
    if (v0 != 0 || v1 != 0) {
      const double yaw = normalize_angle(pr_p(c + DIM * 6, te));
      double sn, cs;
      sincos(yaw, &sn, &cs);
      if (dot2_normalized(v0, v1, cs, sn) < P.cos_yaw_max) return false;
    }
  }
  return true;
}

// validate_primitive (primitive.h:449-470), branch by branch
template <int DIM>
__device__ bool seg_valid(const EnvParams &P, const double *c, double t, int control) {
  switch (control) {
    case MPLX_ACC: return validate_axes<DIM, 1>(c, t, P.v_max);
    case MPLX_JRK: return validate_axes<DIM, 1>(c, t, P.v_max) && validate_axes<DIM, 2>(c, t, P.a_max);
    case MPLX_SNP:
      return validate_axes<DIM, 1>(c, t, P.v_max) && validate_axes<DIM, 2>(c, t, P.a_max) &&
             validate_axes<DIM, 3>(c, t, P.j_max);
    case MPLX_VELxYAW: return validate_yaw_ends<DIM>(P, c, t);
    case MPLX_ACCxYAW: return validate_yaw_ends<DIM>(P, c, t) && validate_axes<DIM, 1>(c, t, P.v_max);
    case MPLX_JRKxYAW:
      return validate_yaw_ends<DIM>(P, c, t) && validate_axes<DIM, 1>(c, t, P.v_max) &&
             validate_axes<DIM, 2>(c, t, P.a_max);
    case MPLX_SNPxYAW:
      return validate_yaw_ends<DIM>(P, c, t) && validate_axes<DIM, 1>(c, t, P.v_max) &&
             validate_axes<DIM, 2>(c, t, P.a_max) && validate_axes<DIM, 3>(c, t, P.j_max);
    default: return true;
  }
}

template <int DIM>
__global__ void __launch_bounds__(128) check_seg_kernel(const __grid_constant__ EnvParams P, CheckArgs A, long long n_wp) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < n_wp; s += (long long)gridDim.x * blockDim.x) {
    const int p = path_of(A.offset, A.n_paths, s);
    const long long b = A.offset[p];
    const int W = (int)(A.offset[p + 1] - b), j = (int)(s - b);
    bool fr = false, va = false;
    if (j + 1 < W) {
      const double *c = A.coeff + s * (DIM + 1) * 6;
      const bool finite = coeff_finite<DIM>(c);
      if (!finite) A.form[p] = 0;  // every writer stores 0
      const double t = A.seg_t[s];
      if (finite && pos_finite(t)) {
        if (A.seg_free) fr = seg_is_free<DIM>(P, c, t);
        if (A.seg_valid) va = seg_valid<DIM>(P, c, t, A.ctl[p]);
      }
    }
    if (A.seg_free) A.seg_free[s] = fr ? 1 : 0;
    if (A.seg_valid) A.seg_valid[s] = va ? 1 : 0;
  }
}

template <int DIM, bool POT>
__global__ void __launch_bounds__(128) check_sample_kernel(const __grid_constant__ EnvParams P, CheckArgs A) {
  constexpr int NC = kCand * DIM;
  constexpr int RW = 4 * DIM + 3;
  constexpr unsigned kAll = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int n_warps = gridDim.x * (blockDim.x >> 5);
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < A.n_paths; p += n_warps) {
    const long long b = A.offset[p];
    const int W = (int)(A.offset[p + 1] - b);
    const int N = A.form[p] ? A.n_pts[p] : 0;
    if (!A.form[p]) {  // a path with a bad segment time or coefficient has no segment results either
      for (int j = lane; j < W; j += 32) {
        if (A.seg_free) A.seg_free[b + j] = 0;
        if (A.seg_valid) A.seg_valid[b + j] = 0;
      }
    }
    if (N == 0) {
      if (lane == 0) {
        A.status[p] = 0;
        A.cost[p] = 0.0;
      }
      continue;
    }
    const double *taus = A.taus + b, *coeff = A.coeff + b * (DIM + 1) * 6;
    const int nl = A.lam ? A.n_lam[p] : 0;
    const double *lam = nl > 0 ? A.lam + b * NC * 7 : nullptr, *lT = A.lam_T + b * NC;
    const bool lam_mono = A.lam_mono[p] != 0;
    const double total = A.total[p], dt = total / N;  // Trajectory::sample(N)
    unsigned carry = 0xffffffffu;  // prev_idx = -1
    double cost = 0.0;
    bool hit = false;
    for (int base = 0; base <= N; base += 32) {
      const int i = base + lane;
      unsigned idx = 0;
      bool inside = false;
      double speed = 0.0;
      if (i <= N) {
        double row[RW];
#pragma unroll
        for (int k = 0; k < RW; k++) row[k] = 0.0;
        traj_row<DIM>(taus, W - 1, coeff, lam, lT, nl, lam_mono, total, i * dt, row);
        int pn[DIM];
        inside = true;
#pragma unroll
        for (int a = 0; a < DIM; a++) {
          pn[a] = float_to_int(row[a], P.origin[a], P.res);
          inside = inside && (unsigned)pn[a] < (unsigned)P.mdim[a];
        }
        // getIndex before any bounds test, int arithmetic wrapping as on the reference's targets
        idx = (unsigned)pn[0] + (unsigned)P.mdim[0] * (unsigned)pn[1];
        if (DIM == 3) idx += (unsigned)P.mdim[0] * (unsigned)P.mdim[1] * (unsigned)pn[DIM - 1];
        if (POT) {  // Vecf::norm: Eigen's a0 + a1, a0 + (a1 + a2)
          const double *v = row + DIM;
          speed = DIM == 2 ? sqrt(v[0] * v[0] + v[1] * v[1]) : sqrt(v[0] * v[0] + (v[1] * v[1] + v[DIM - 1] * v[DIM - 1]));
        }
      }
      unsigned prev = __shfl_up_sync(kAll, idx, 1);
      if (lane == 0) prev = carry;
      carry = __shfl_sync(kAll, idx, 31);
      const bool counted = i <= N && idx != prev;
      bool bad = false, has_term = false;
      double term = 0.0;
      if (counted) {
        if (!inside) {
          bad = true;
        } else if (POT) {
          const int pv = __ldg(P.pot + idx);
          if (pv >= 100) bad = true;
          else if (pv > 0) {
            term = P.pot_w * pv + P.grad_w * speed;
            has_term = true;
          }
        } else {
          bad = (__ldg(P.occ_bits + (idx >> 5)) >> (idx & 31)) & 1u;
        }
      }
      if (__ballot_sync(kAll, bad)) {
        hit = true;
        break;
      }
      if (POT) {
        for (unsigned m = __ballot_sync(kAll, has_term); m; m &= m - 1) cost = cost + __shfl_sync(kAll, term, __ffs(m) - 1);
      }
    }
    if (lane == 0) {
      A.status[p] = 1;
      A.cost[p] = hit ? (double)INFINITY : cost;
    }
  }
}

cudaError_t launch_check(int dim, bool pot, const EnvParams &P, const CheckArgs &A, long long n_wp, cudaStream_t st,
                         int *launches) {
  return with_dim(dim, [&](auto DIM) {
    if (cudaError_t e = launch(check_path_kernel<DIM>, A.n_paths, false, st, launches, P, A)) return e;
    if (cudaError_t e = launch(check_seg_kernel<DIM>, n_wp, true, st, launches, P, A, n_wp)) return e;
    return with_bool(pot, [&](auto POT) {
      return launch(check_sample_kernel<DIM, POT>, 32LL * A.n_paths, true, st, launches, P, A);
    });
  });
}

}  // namespace
}  // namespace mplx

extern "C" int mplx_traj_check(mplx_ctx *c, int n_paths, const int64_t *offset, const double *seg_t,
                               const double *coeff, const uint8_t *control, const double *total_t,
                               const int32_t *n_lambda, const double *lambda, mplx_traj_check_out *out) {
  if (int r = mplx_bind(c)) return r;
  if (!c->has_map) return fail(MPLX_ERR_ARG, "no map: call mplx_set_map first");
  if (!c->has_params) return fail(MPLX_ERR_ARG, "no params: call mplx_set_params first");
  long long n_wp = 0;
  if (int r = mplx::check_batch(n_paths, offset, out && out->status && out->cost, seg_t && coeff, false, 0, n_wp))
    return r;
  if (out->seg_valid && !control) return fail(MPLX_ERR_ARG, "seg_valid without control");
  const bool scaled = lambda != nullptr;
  if ((total_t != nullptr) != scaled || (n_lambda != nullptr) != scaled)
    return fail(MPLX_ERR_ARG, "total_t, n_lambda and lambda go together");
  const int dim = c->dim;
  const long long NC = (long long)mplx::kCand * dim;
  if (scaled)
    for (int p = 0; p < n_paths; p++)
      if (n_lambda[p] < 0 || n_lambda[p] > (offset[p + 1] - offset[p]) * NC)
        return fail(MPLX_ERR_ARG, "n_lambda[%d] = %d outside [0, %lld]", p, n_lambda[p], (offset[p + 1] - offset[p]) * NC);
  out->seconds = 0.0;
  if (n_paths == 0) return MPLX_OK;
  TrajBufs &B = c->tb;
  const size_t nw = (size_t)std::max<long long>(n_wp, 1);
  CU(B.offset.reserve(n_paths + 1)); CU(B.status.reserve(n_paths)); CU(B.mono.reserve(n_paths));
  CU(B.n_pts.reserve(n_paths)); CU(B.form.reserve(n_paths)); CU(B.total.reserve(n_paths)); CU(B.cost.reserve(n_paths));
  CU(B.seg_t.reserve(nw)); CU(B.taus.reserve(nw)); CU(B.coeff.reserve(nw * (dim + 1) * 6));
  if (out->seg_free) CU(B.seg_free.reserve(nw));
  if (out->seg_valid) {
    CU(B.seg_valid.reserve(nw));
    CU(B.ctl.reserve(n_paths));
  }
  if (scaled) {
    CU(B.par.reserve(n_paths)); CU(B.n_knot.reserve(n_paths));
    CU(B.lam.reserve(nw * NC * 7)); CU(B.lam_T.reserve(nw * NC + 1));
  }
  cudaStream_t st = c->stream;
  CU(cudaMemcpyAsync(B.offset.p, offset, sizeof(int64_t) * (n_paths + 1), cudaMemcpyHostToDevice, st));
  if (n_wp > 0) {
    CU(cudaMemcpyAsync(B.seg_t.p, seg_t, sizeof(double) * n_wp, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(B.coeff.p, coeff, sizeof(double) * n_wp * (dim + 1) * 6, cudaMemcpyHostToDevice, st));
  }
  if (out->seg_valid) CU(cudaMemcpyAsync(B.ctl.p, control, (size_t)n_paths, cudaMemcpyHostToDevice, st));
  if (scaled) {
    CU(cudaMemcpyAsync(B.par.p, total_t, sizeof(double) * n_paths, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(B.n_knot.p, n_lambda, sizeof(int32_t) * n_paths, cudaMemcpyHostToDevice, st));
    if (n_wp > 0) CU(cudaMemcpyAsync(B.lam.p, lambda, sizeof(double) * n_wp * NC * 7, cudaMemcpyHostToDevice, st));
  }
  mplx::CheckArgs A{n_paths, B.offset.p, B.seg_t.p, B.coeff.p, scaled ? B.par.p : nullptr, scaled ? B.lam.p : nullptr,
                    scaled ? B.n_knot.p : nullptr, out->seg_valid ? B.ctl.p : nullptr, B.status.p, B.n_pts.p, B.form.p,
                    B.mono.p, B.taus.p, B.lam_T.p, B.total.p, B.cost.p, out->seg_free ? B.seg_free.p : nullptr,
                    out->seg_valid ? B.seg_valid.p : nullptr};
  TimedRun timed;
  CU(timed.run(st, c->launches, [&](int *launches) {
    return mplx::launch_check(dim, c->P.pot != nullptr, c->P, A, n_wp, st, launches);
  }));
  CU(cudaMemcpyAsync(out->status, B.status.p, sizeof(int32_t) * n_paths, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(out->cost, B.cost.p, sizeof(double) * n_paths, cudaMemcpyDeviceToHost, st));
  if (n_wp > 0 && out->seg_free) CU(cudaMemcpyAsync(out->seg_free, B.seg_free.p, (size_t)n_wp, cudaMemcpyDeviceToHost, st));
  if (n_wp > 0 && out->seg_valid) CU(cudaMemcpyAsync(out->seg_valid, B.seg_valid.p, (size_t)n_wp, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(timed.seconds(&out->seconds));
  return MPLX_OK;
}
