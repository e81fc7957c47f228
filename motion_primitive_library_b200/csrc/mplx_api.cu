// mplx_api.cu — the C ABI of include/mplx.h: context, HBM staging of the static per-plan
// data, and the host-buffer / device-buffer expansion entry points.
//
// No CPU fallback lives here: without a usable CUDA device every compute call fails.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <vector>

#include "../../include/mplx.h"
#include "mplx_internal.h"
#include "mplx_pack.cuh"

namespace mplx {
thread_local char g_err[512] = "";
int fail(int code, const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
  return code;
}
}  // namespace mplx
using mplx::g_err;

int mplx_bind(mplx_ctx *ctx) {
  if (!ctx) return fail(MPLX_ERR_ARG, "null ctx");
  CU(cudaSetDevice(ctx->device));
  return MPLX_OK;
}

// L2 persisting carve-out for the bitmap pairs (up to what the device grants): see launch_expand_fxn.  Both halves
// when they fit it; otherwise the occupancy half, which every sample reads, and not the summary half, which only
// uncertain samples read (a window larger than the carve-out thrashes it).  Reserved only while the fixed-point
// kernels can run (fx_supported: a map without a potential field, no yaw control, occ2 within its address
// range); otherwise none is set aside: the set-aside takes L2 from the kernels that do run (cfg4, which never
// reads occ2, was 1.5 % slower per step with 22.8 MiB set aside than with 16 MiB).
void mplx::size_l2_window(mplx_ctx *c) {
  size_t bytes = 0;
  int maxp = 0, maxw = 0;
  if (c->has_map && !c->has_pot && (c->P.control & 16) == 0 && c->P.occ2_sum <= (1u << 27)) {
    cudaDeviceGetAttribute(&maxp, cudaDevAttrMaxPersistingL2CacheSize, c->device);
    cudaDeviceGetAttribute(&maxw, cudaDevAttrMaxAccessPolicyWindowSize, c->device);
    const size_t half = (size_t)c->P.occ2_sum * sizeof(uint32_t);
    if (maxp > 0 && maxw > 0) bytes = 2 * half <= (size_t)maxp ? 2 * half : half;
  }
  const size_t want = bytes < (size_t)maxp ? bytes : (size_t)maxp;
  if (want != c->l2_persist) {
    if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) != cudaSuccess) {
      cudaGetLastError();
      bytes = 0;
    }
    c->l2_persist = want;
  }
  c->occ2_window = bytes < (size_t)maxw ? bytes : (size_t)maxw;
}

static void refresh_params(mplx_ctx *c) {
  c->P.map = c->has_map ? c->map.p : nullptr;
  c->P.pot = c->has_pot ? c->pot.p : nullptr;
  c->P.region_bits = c->has_region ? c->region.p : nullptr;
  c->P.U = c->U.p;
  c->P.stats = c->stats_on ? c->stats.p : nullptr;
  c->P.occ_bits = c->has_map ? c->occ.p : nullptr;
  c->P.occ2 = c->has_map ? c->occ2.p : nullptr;
  mplx::size_l2_window(c);
  c->P.occ2_bytes = c->has_map ? c->occ2_window : 0;
  c->P.prow = c->prow.p;
  c->P.row_u = c->row_u.p;
  c->P.row_axis = c->row_axis.p;
  c->P.n_rows = c->n_rows;
  c->P.ttab = c->ttab.p;
  c->P.tcount = c->tcount.p;
  c->P.tdt = c->tdt.p;
  // largest sample count n the flat phase will meet: validated primitives have
  // max_vel <= v_max (primitive.h:482-496), so n = max(5, ceil(max_v*T/res)) (env_map.h:95)
  // is bounded; VEL control and v_max <= 0 are unbounded -> whole table.
  int maxn = mplx::kNMax;
  if (c->has_map && c->has_params && (c->P.control & 15) != MPLX_VEL && c->P.v_max > 0) {
    const double nb = ceil(c->P.v_max * c->P.T / c->P.res);
    if (nb < (double)mplx::kNMax) maxn = nb < 5 ? 5 : (int)nb;
  }
  c->P.maxn = maxn;
}

extern "C" {

const char *mplx_last_error(void) { return g_err; }

const char *mplx_build_info(void) {
  return "libmplx sm_90a; nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false; "
         "IEEE double, no CPU fallback";
}

int mplx_create(int dim, int device, mplx_ctx **out) {
  if (!out) return fail(MPLX_ERR_ARG, "out is null");
  *out = nullptr;
  if (dim != 2 && dim != 3) return fail(MPLX_ERR_ARG, "dim must be 2 or 3, got %d", dim);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(MPLX_ERR_CUDA, "no CUDA device available (%s); libmplx has no CPU fallback",
                e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  }
  if (device < 0 || device >= ndev) return fail(MPLX_ERR_ARG, "device %d out of range [0,%d)", device, ndev);
  CU(cudaSetDevice(device));
  mplx_ctx *c = new (std::nothrow) mplx_ctx();
  if (!c) return fail(MPLX_ERR_ALLOC, "host allocation failed");
  c->dim = dim;
  c->device = device;
  if (const char *k = getenv("MPLX_KERNEL")) {  // diagnostics: initial mplx_set_kernel value
    const int w = atoi(k);
    if (w >= 0 && w <= 5) c->kernel = w;
  }
  memset(&c->P, 0, sizeof c->P);
  c->P.dim = dim;
  e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    delete c;
    return fail(MPLX_ERR_CUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(e));
  }
  e = c->stats.reserve(2);
  if (e != cudaSuccess) {
    cudaStreamDestroy(c->stream);
    delete c;
    return fail(MPLX_ERR_ALLOC, "cudaMalloc failed: %s", cudaGetErrorString(e));
  }
  *out = c;
  return MPLX_OK;
}

int mplx_destroy(mplx_ctx *c) {
  if (!c) return MPLX_OK;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  c->map.release(); c->pot.release(); c->region.release(); c->U.release(); c->stats.release();
  c->prow.release(); c->row_axis.release(); c->row_u.release();
  c->occ.release(); c->occ2.release(); c->ttab.release(); c->tcount.release(); c->tdt.release();
  for (int b = 0; b < kPackBufs; b++) c->cb[b].release();
  if (c->d2h_stream) cudaStreamDestroy(c->d2h_stream);
  c->eb.release(); c->fxq.release(); c->ub.release(); c->sb.release(); c->tun.release(); c->tb.release();
  c->d_nodes.release(); c->d_succ.release(); c->d_count.release(); c->d_action.release();
  c->d_lattice.release(); c->d_cost.release(); c->d_key.release();
  c->h_nodes.release(); c->h_succ.release(); c->h_count.release(); c->h_action.release();
  c->h_lattice.release(); c->h_cost.release(); c->h_key.release();
  cudaStreamDestroy(c->stream);
  delete c;
  return MPLX_OK;
}

int mplx_set_map(mplx_ctx *c, const int8_t *data, const int32_t *dim, const double *origin, double res) {
  if (int r = mplx_bind(c)) return r;
  if (!data || !dim || !origin) return fail(MPLX_ERR_ARG, "null argument");
  if (!(res > 0)) return fail(MPLX_ERR_ARG, "res must be > 0");
  size_t nvox = 1;
  for (int k = 0; k < c->dim; k++) {
    if (dim[k] <= 0) return fail(MPLX_ERR_ARG, "dim[%d] = %d", k, dim[k]);
    nvox *= (size_t)dim[k];
  }
  if (nvox >= (size_t)1 << 31) return fail(MPLX_ERR_ARG, "grid has %zu cells; getIndex is int32 (map_util.h:34-41)", nvox);
  CU(cudaStreamSynchronize(c->stream));
  CU(c->map.reserve(nvox));
  CU(cudaMemcpyAsync(c->map.p, data, nvox, cudaMemcpyHostToDevice, c->stream));
  CU(c->occ.reserve((nvox + 31) / 32));
  CU(mplx::launch_pack_bits(c->map.p, nvox, c->occ.p, true, c->stream));
  const int nz = c->dim == 3 ? dim[2] : 1;
  const size_t npairs = mplx::occ2_guard_pair_count(c->dim, dim[0], dim[1], nz);
  CU(c->occ2.reserve(2 * npairs));
  CU(mplx::launch_pack_occ2(c->occ.p, nvox, c->dim, dim[0], dim[1], nz, c->occ2.p, c->stream));
  c->launches += 2;
  CU(cudaStreamSynchronize(c->stream));
  c->nvox = nvox;
  for (int k = 0; k < 3; k++) {
    c->P.mdim[k] = k < c->dim ? dim[k] : 1;
    c->P.origin[k] = k < c->dim ? origin[k] : 0.0;
    c->P.dimd[k] = (double)c->P.mdim[k];
  }
  mplx::occ2_sep_terms(c->dim, dim[0], dim[1], mplx::kFxHiBase, c->P.occ2_e, c->P.occ2_k0);
  c->P.occ2_sum = npairs < ((size_t)1 << 32) ? (unsigned)npairs : ~0u;  // ~0u: beyond the fixed-point kernels (fx_supported)
  c->P.res = res;
  c->P.rinv = 1.0 / res;
  c->has_map = true;
  c->has_pot = false;
  c->has_region = false;
  c->tun.release();  // the per-query tunnels go with the ctx-wide region
  refresh_params(c);
  return MPLX_OK;
}

int mplx_set_potential(mplx_ctx *c, const int8_t *data, double pw, double gw) {
  if (int r = mplx_bind(c)) return r;
  if (!c->has_map) return fail(MPLX_ERR_ARG, "mplx_set_map must be called first");
  c->P.pot_w = pw;
  c->P.grad_w = gw;
  if (!data) {
    c->has_pot = false;
  } else {
    CU(cudaStreamSynchronize(c->stream));
    CU(c->pot.reserve(c->nvox));
    CU(cudaMemcpyAsync(c->pot.p, data, c->nvox, cudaMemcpyHostToDevice, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    c->has_pot = true;
  }
  refresh_params(c);
  return MPLX_OK;
}

int mplx_set_potential_weights(mplx_ctx *c, double pw, double gw) {
  if (int r = mplx_bind(c)) return r;
  c->P.pot_w = pw;
  c->P.grad_w = gw;
  return MPLX_OK;
}

int mplx_set_search_region(mplx_ctx *c, const uint8_t *in_region) {
  if (int r = mplx_bind(c)) return r;
  if (!c->has_map) return fail(MPLX_ERR_ARG, "mplx_set_map must be called first");
  if (!in_region) {
    c->has_region = false;
  } else {
    CU(cudaStreamSynchronize(c->stream));
    DevBuf<uint8_t> tmp;
    CU(tmp.reserve(c->nvox));
    cudaError_t e = cudaMemcpyAsync(tmp.p, in_region, c->nvox, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = c->region.reserve((c->nvox + 31) / 32);
    if (e == cudaSuccess) e = mplx::launch_pack_bits((const int8_t *)tmp.p, c->nvox, c->region.p, false, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    tmp.release();
    CU(e);
    c->launches++;
    c->has_region = true;
  }
  refresh_params(c);
  return MPLX_OK;
}

int mplx_set_params(mplx_ctx *c, int control, double T, double w, double wyaw, double v_max,
                    double a_max, double j_max, double yaw_max, const double *U, int nU, int udim) {
  if (int r = mplx_bind(c)) return r;
  const int base = control & 15;
  if ((control & ~31) || (base != MPLX_VEL && base != MPLX_ACC && base != MPLX_JRK && base != MPLX_SNP))
    return fail(MPLX_ERR_ARG, "control 0x%x is not a Control::Control value (control.h:10-20)", control);
  const bool yaw = control & 16;
  if (!U || nU <= 0 || nU > mplx::kMaxU) return fail(MPLX_ERR_ARG, "need 1 <= nU <= %d controls", mplx::kMaxU);
  if (udim != c->dim + (yaw ? 1 : 0))
    return fail(MPLX_ERR_ARG, "udim %d must be dim%s = %d for control 0x%x", udim, yaw ? "+1" : "", c->dim + (yaw ? 1 : 0), control);
  if (!(T > 0)) return fail(MPLX_ERR_ARG, "T (dt_) must be > 0");
  CU(cudaStreamSynchronize(c->stream));
  CU(c->U.reserve((size_t)nU * udim));
  CU(cudaMemcpyAsync(c->U.p, U, sizeof(double) * nU * udim, cudaMemcpyHostToDevice, c->stream));
  {
    // per-axis value tables: distinct values (bitwise) of every position axis of U, in order of appearance
    std::vector<unsigned char> prow((size_t)nU * 3, 0), row_axis;
    std::vector<double> row_u;
    bool fits = true;
    for (int a = 0; a < c->dim && fits; a++) {
      const size_t first = row_u.size();
      for (int i = 0; i < nU; i++) {
        const double v = U[(size_t)i * udim + a];
        size_t r = first;
        for (; r < row_u.size(); r++)
          if (memcmp(&row_u[r], &v, sizeof v) == 0) break;
        if (r == row_u.size()) {
          if (row_u.size() >= 255) { fits = false; break; }
          row_u.push_back(v);
          row_axis.push_back((unsigned char)a);
        }
        prow[(size_t)i * 3 + a] = (unsigned char)r;
      }
    }
    c->n_rows = 0;
    if (fits) {
      CU(c->prow.reserve(prow.size()));
      CU(c->row_u.reserve(row_u.size()));
      CU(c->row_axis.reserve(row_axis.size()));
      CU(cudaMemcpyAsync(c->prow.p, prow.data(), prow.size(), cudaMemcpyHostToDevice, c->stream));
      CU(cudaMemcpyAsync(c->row_u.p, row_u.data(), sizeof(double) * row_u.size(), cudaMemcpyHostToDevice, c->stream));
      CU(cudaMemcpyAsync(c->row_axis.p, row_axis.data(), row_axis.size(), cudaMemcpyHostToDevice, c->stream));
      CU(cudaStreamSynchronize(c->stream));  // the vectors die at the end of this block
      c->n_rows = (int)row_u.size();
    }
  }
  CU(c->ttab.reserve((size_t)(mplx::kNMax + 1) * mplx::kTStride + 8));  // + padding: units read 4 times at once
  CU(c->tcount.reserve(mplx::kNMax + 1));
  CU(c->tdt.reserve(mplx::kNMax + 1));
  CU(cudaMemsetAsync(c->ttab.p, 0, sizeof(double) * ((size_t)(mplx::kNMax + 1) * mplx::kTStride + 8), c->stream));
  CU(mplx::launch_build_ttab(T, c->ttab.p, c->tcount.p, c->tdt.p, c->stream));
  c->launches++;
  CU(cudaStreamSynchronize(c->stream));
  c->P.control = control;
  c->P.nU = nU;
  c->P.udim = udim;
  c->P.T = T;
  c->P.w = w;
  c->P.wyaw = wyaw;
  c->P.v_max = v_max;
  c->P.a_max = a_max;
  c->P.j_max = j_max;
  c->P.yaw_max = yaw_max;
  c->P.cos_yaw_max = cos(yaw_max);  // host libm, as the reference's cos(my) (primitive.h:521)
  c->has_params = true;
  refresh_params(c);
  return MPLX_OK;
}

int mplx_check_ready(mplx_ctx *c, int n_nodes) {
  if (!c->has_map) return fail(MPLX_ERR_ARG, "no map: call mplx_set_map first");
  if (!c->has_params) return fail(MPLX_ERR_ARG, "no params: call mplx_set_params first");
  if (n_nodes < 0) return fail(MPLX_ERR_ARG, "n_nodes < 0");
  if ((size_t)n_nodes * c->P.nU >= ((size_t)1 << 31)) return fail(MPLX_ERR_ARG, "batch too large");
  return MPLX_OK;
}
static int check_ready(mplx_ctx *c, int n_nodes, const mplx_succ_out *out) {
  if (int r = mplx_check_ready(c, n_nodes)) return r;
  if (!out || !out->count) return fail(MPLX_ERR_ARG, "out->count is required");
  return MPLX_OK;
}

int mplx_expand_device(mplx_ctx *c, const void *d_nodes, int n_nodes, const mplx_succ_out *out, void *stream) {
  if (int r = mplx_bind(c)) return r;
  if (int r = check_ready(c, n_nodes, out)) return r;
  if (n_nodes == 0) return MPLX_OK;
  if (!d_nodes) return fail(MPLX_ERR_ARG, "d_nodes is null");
  cudaStream_t st = stream ? (cudaStream_t)stream : c->stream;
  if (c->stats_on) CU(cudaMemsetAsync(c->stats.p, 0, 2 * sizeof(unsigned long long), st));
  CU(c->fxq.reserve((size_t)n_nodes * c->P.nU));
  int launches = 0;
  CU(mplx::launch_expand(c->P, (const mplx_waypoint *)d_nodes, n_nodes, *out, st, c->kernel, &c->fxq.view, &launches));
  c->launches += launches;
  if (c->stats_on)
    CU(cudaMemcpyAsync(c->last_stats, c->stats.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  return MPLX_OK;
}

int mplx_expand(mplx_ctx *c, const mplx_waypoint *nodes, int n_nodes, const mplx_succ_out *out) {
  if (int r = mplx_bind(c)) return r;
  if (int r = check_ready(c, n_nodes, out)) return r;
  if (n_nodes == 0) return MPLX_OK;
  if (!nodes) return fail(MPLX_ERR_ARG, "nodes is null");
  const int nU = c->P.nU;
  // chunk so that staging stays bounded (~1M successor slots per chunk)
  int chunk = (1 << 20) / nU;
  if (chunk < 1) chunk = 1;
  if (chunk > n_nodes) chunk = n_nodes;
  const size_t slots = (size_t)chunk * nU;
  cudaStream_t st = c->stream;

  CU(c->d_nodes.reserve(chunk));
  CU(c->d_count.reserve(chunk));
  if (out->succ) CU(c->d_succ.reserve(slots));
  if (out->cost) CU(c->d_cost.reserve(slots));
  if (out->action) CU(c->d_action.reserve(slots));
  if (out->key) CU(c->d_key.reserve(slots));
  if (out->lattice) CU(c->d_lattice.reserve(slots * MPLX_LATTICE_MAX));

  const bool pin_nodes = is_pinned(nodes), pin_count = is_pinned(out->count), pin_succ = is_pinned(out->succ),
             pin_cost = is_pinned(out->cost), pin_action = is_pinned(out->action), pin_key = is_pinned(out->key),
             pin_lat = is_pinned(out->lattice);
  if (!pin_nodes) CU(c->h_nodes.reserve(chunk));
  if (!pin_count) CU(c->h_count.reserve(chunk));
  if (out->succ && !pin_succ) CU(c->h_succ.reserve(slots));
  if (out->cost && !pin_cost) CU(c->h_cost.reserve(slots));
  if (out->action && !pin_action) CU(c->h_action.reserve(slots));
  if (out->key && !pin_key) CU(c->h_key.reserve(slots));
  if (out->lattice && !pin_lat) CU(c->h_lattice.reserve(slots * MPLX_LATTICE_MAX));

  // Small batches (the one-node get_succ of a planner without speculation, a few dozen nodes with it): the
  // kernel reads the nodes from, and writes the successors to, pinned host memory directly — one launch and
  // one wait instead of one copy in, up to six copies out and the wait.  (For large batches SM stores over
  // PCIe lose against the copy engines: mplx_packed.cu.)
  static const bool no_zero_copy = getenv("MPLX_NO_ZERO_COPY") != nullptr;  // tuning / A-B
  if (!no_zero_copy && !c->stats_on && (size_t)n_nodes * nU <= 4096) {
    const int m = n_nodes;
    const size_t sm = (size_t)m * nU;
    const mplx_waypoint *src = nodes;
    if (!pin_nodes) {
      memcpy(c->h_nodes.p, nodes, sizeof(mplx_waypoint) * m);
      src = c->h_nodes.p;
    }
    mplx_succ_out d;
    d.count = pin_count ? out->count : c->h_count.p;
    d.succ = out->succ ? (pin_succ ? out->succ : c->h_succ.p) : nullptr;
    d.cost = out->cost ? (pin_cost ? out->cost : c->h_cost.p) : nullptr;
    d.action = out->action ? (pin_action ? out->action : c->h_action.p) : nullptr;
    d.key = out->key ? (pin_key ? out->key : c->h_key.p) : nullptr;
    d.lattice = out->lattice ? (pin_lat ? out->lattice : c->h_lattice.p) : nullptr;
    CU(c->fxq.reserve(sm));
    int launches = 0;
    CU(mplx::launch_expand(c->P, src, m, d, st, c->kernel, &c->fxq.view, &launches));
    c->launches += launches;
    CU(cudaStreamSynchronize(st));
    if (!pin_count) memcpy(out->count, c->h_count.p, sizeof(int32_t) * m);
    if (out->succ && !pin_succ) memcpy(out->succ, c->h_succ.p, sizeof(mplx_waypoint) * sm);
    if (out->cost && !pin_cost) memcpy(out->cost, c->h_cost.p, sizeof(double) * sm);
    if (out->action && !pin_action) memcpy(out->action, c->h_action.p, sizeof(int32_t) * sm);
    if (out->key && !pin_key) memcpy(out->key, c->h_key.p, sizeof(uint64_t) * sm);
    if (out->lattice && !pin_lat) memcpy(out->lattice, c->h_lattice.p, sizeof(int32_t) * sm * MPLX_LATTICE_MAX);
    return MPLX_OK;
  }

  unsigned long long acc_stats[2] = {0, 0};
  for (int off = 0; off < n_nodes; off += chunk) {
    const int m = n_nodes - off < chunk ? n_nodes - off : chunk;
    const size_t so = (size_t)off * nU, sm = (size_t)m * nU;
    const mplx_waypoint *src = nodes + off;
    if (!pin_nodes) {
      memcpy(c->h_nodes.p, src, sizeof(mplx_waypoint) * m);
      src = c->h_nodes.p;
    }
    CU(cudaMemcpyAsync(c->d_nodes.p, src, sizeof(mplx_waypoint) * m, cudaMemcpyHostToDevice, st));
    mplx_succ_out d;
    d.count = c->d_count.p;
    d.succ = out->succ ? c->d_succ.p : nullptr;
    d.cost = out->cost ? c->d_cost.p : nullptr;
    d.action = out->action ? c->d_action.p : nullptr;
    d.key = out->key ? c->d_key.p : nullptr;
    d.lattice = out->lattice ? c->d_lattice.p : nullptr;
    if (c->stats_on) CU(cudaMemsetAsync(c->stats.p, 0, 2 * sizeof(unsigned long long), st));
    CU(c->fxq.reserve((size_t)m * nU));
    int launches = 0;
    CU(mplx::launch_expand(c->P, c->d_nodes.p, m, d, st, c->kernel, &c->fxq.view, &launches));
    c->launches += launches;
    if (c->stats_on)
      CU(cudaMemcpyAsync(c->last_stats, c->stats.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
#define D2H(field, T, mult, pinflag, hbuf)                                                              \
  if (out->field) {                                                                                    \
    T *dst = pinflag ? out->field + so * (mult) : hbuf.p;                                              \
    CU(cudaMemcpyAsync(dst, d.field, sizeof(T) * sm * (mult), cudaMemcpyDeviceToHost, st));             \
  }
    {
      int32_t *dst = pin_count ? out->count + off : c->h_count.p;
      CU(cudaMemcpyAsync(dst, d.count, sizeof(int32_t) * m, cudaMemcpyDeviceToHost, st));
    }
    D2H(succ, mplx_waypoint, 1, pin_succ, c->h_succ)
    D2H(cost, double, 1, pin_cost, c->h_cost)
    D2H(action, int32_t, 1, pin_action, c->h_action)
    D2H(key, uint64_t, 1, pin_key, c->h_key)
    D2H(lattice, int32_t, MPLX_LATTICE_MAX, pin_lat, c->h_lattice)
#undef D2H
    CU(cudaStreamSynchronize(st));
    if (!pin_count) memcpy(out->count + off, c->h_count.p, sizeof(int32_t) * m);
    if (out->succ && !pin_succ) memcpy(out->succ + so, c->h_succ.p, sizeof(mplx_waypoint) * sm);
    if (out->cost && !pin_cost) memcpy(out->cost + so, c->h_cost.p, sizeof(double) * sm);
    if (out->action && !pin_action) memcpy(out->action + so, c->h_action.p, sizeof(int32_t) * sm);
    if (out->key && !pin_key) memcpy(out->key + so, c->h_key.p, sizeof(uint64_t) * sm);
    if (out->lattice && !pin_lat)
      memcpy(out->lattice + so * MPLX_LATTICE_MAX, c->h_lattice.p, sizeof(int32_t) * sm * MPLX_LATTICE_MAX);
    if (c->stats_on) {
      acc_stats[0] += c->last_stats[0];
      acc_stats[1] += c->last_stats[1];
    }
  }
  if (c->stats_on) {
    c->last_stats[0] = acc_stats[0];
    c->last_stats[1] = acc_stats[1];
  }
  return MPLX_OK;
}

int mplx_set_kernel(mplx_ctx *c, int which) {
  if (!c) return fail(MPLX_ERR_ARG, "null ctx");
  if (which < 0 || which > 5)
    return fail(MPLX_ERR_ARG, "which must be 0 (auto), 1 (sequential), 2 (register), 3 (flat), 4 (dealing) or 5 (fixed-point)");
  c->kernel = which;
  return MPLX_OK;
}

int mplx_sync(mplx_ctx *c) {
  if (int r = mplx_bind(c)) return r;
  CU(cudaStreamSynchronize(c->stream));
  return MPLX_OK;
}

int64_t mplx_launch_count(const mplx_ctx *c) { return c ? c->launches : 0; }

int mplx_enable_stats(mplx_ctx *c, int on) {
  if (int r = mplx_bind(c)) return r;
  c->stats_on = on != 0;
  refresh_params(c);
  return MPLX_OK;
}

int mplx_last_stats(mplx_ctx *c, int64_t *samples, int64_t *successors) {
  if (int r = mplx_bind(c)) return r;
  CU(cudaStreamSynchronize(c->stream));
  if (samples) *samples = (int64_t)c->last_stats[0];
  if (successors) *successors = (int64_t)c->last_stats[1];
  return MPLX_OK;
}

void *mplx_stream(mplx_ctx *c) { return c ? (void *)c->stream : nullptr; }

void *mplx_host_alloc(size_t bytes) {
  void *p = nullptr;
  if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    fail(MPLX_ERR_ALLOC, "cudaHostAlloc(%zu) failed", bytes);
    return nullptr;
  }
  return p;
}

void mplx_host_free(void *p) {
  if (p) cudaFreeHost(p);
}

}  // extern "C"
