// mplx_dispatch.h — the run-time plan -> kernel template parameters mapping of every launcher (host only).
// Each with_* calls f with the value as a std::integral_constant, so that f can use it as a template
// argument and rule instantiations out with `if constexpr`; f returns a cudaError_t.
#pragma once
#include <cuda_runtime.h>

#include <type_traits>

#include "../../include/mplx.h"

namespace mplx {

template <int V>
using Int = std::integral_constant<int, V>;

template <class F>
cudaError_t with_dim(int dim, F &&f) {
  switch (dim) {
    case 2: return f(Int<2>());
    case 3: return f(Int<3>());
  }
  return cudaErrorInvalidValue;
}

// polynomial order of the position axes of a Control::Control value (control.h:10-20), yaw bit aside
template <class F>
cudaError_t with_order(int control, F &&f) {
  switch (control & 15) {
    case MPLX_VEL: return f(Int<1>());
    case MPLX_ACC: return f(Int<2>());
    case MPLX_JRK: return f(Int<3>());
    case MPLX_SNP: return f(Int<4>());
  }
  return cudaErrorInvalidValue;
}

template <class F>
cudaError_t with_bool(bool b, F &&f) {
  return b ? f(std::true_type()) : f(std::false_type());
}

}  // namespace mplx
