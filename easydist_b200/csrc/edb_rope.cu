// Rotary position embedding (RoPE) of the Llama attention, forward and backward, for the sharded-op
// kernel dispatch of libedb.so.
//
// Traced, RoPE of a [B, H, T, hd] tensor is a chain of about ten elementwise ATen ops (slices, four
// multiplies by the [T, hd/2] cos / sin tables, sub, add, cat; the backward adds a neg, two
// slice_backward zero fills and an add, and the projection GEMMs then need a transpose + clone).  With
// x1, x2 the two halves of the head dim, every form of the chain computes, with fp32 arithmetic and T()
// the rounding to the tensor dtype,
//   y1 = T(T(x1*c) - T(x2*s')),   y2 = T(T(x2*c) + T(x1*s')),   s' = s (forward) or -s (backward)
// (the backward also turns a -0 into +0, as its zero-filled adds do).  Every rounding point is kept:
// the products and sums use __fmul_rn / __fadd_rn / __fsub_rn, so the compiler cannot contract them
// into FMAs, and the result is bit-identical to the ATen chain.  One read of x, one write of y:
// 2*n*sizeof(T) bytes; the tables are [T, half] and broadcast over (b, h), so they stay in L2.
//
// x and y are addressed through (b, h, t) element strides (last dimension contiguous), so the kernel
// reads the transposed view of the projection output directly and writes either the [B, H, T, hd]
// layout attention reads or the [B, T, H, hd] layout the projection GEMMs of the backward read.
// Work: blockIdx.y walks (b, h); the threads of blockIdx.x walk (t, j), j a group of EPV elements of
// the half (16-byte vectors when every pointer, stride and `half` allow it, else EPV = 1).
#include <cuda_bf16.h>

#include "edb_internal.cuh"
#include "edb_vec.cuh"

namespace edb {

constexpr int kRopeMaxHalf = 256;  // head dim <= 512

struct RopeStrides {
  int64_t x0, x1, x2, y0, y1, y2, tab;
};

template <typename T, int EPV>
__device__ __forceinline__ void rope_ld(const T* p, float* f) {
  if constexpr (EPV == 1) f[0] = VecT<T>::ld(p);
  else VecT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(p)), f);
}

template <typename T, int EPV>
__device__ __forceinline__ void rope_st(T* p, const float* f) {
  if constexpr (EPV == 1) VecT<T>::st(p, f[0]);
  else *reinterpret_cast<uint4*>(p) = VecT<T>::pack(f);
}

template <typename T, int EPV>
__global__ void __launch_bounds__(256)
    k_rope(T* __restrict__ y, const T* __restrict__ x, const T* __restrict__ cs,
           const T* __restrict__ sn, int64_t bh_n, int H, int per_bh, int nvh, int half,
           RopeStrides st, int inverse) {
  using V = VecT<T>;
  for (int64_t bh = blockIdx.y; bh < bh_n; bh += gridDim.y) {
    const int64_t b = bh / H, h = bh - b * H;
    const T* xb = x + b * st.x0 + h * st.x1;
    T* yb = y + b * st.y0 + h * st.y1;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_bh; i += gridDim.x * blockDim.x) {
      const int t = i / nvh, j = (i - t * nvh) * EPV;
      const T* xr = xb + t * st.x2 + j;
      T* yr = yb + t * st.y2 + j;
      const int64_t tj = t * st.tab + j;
      float x1[EPV], x2[EPV], c[EPV], s[EPV], y1[EPV], y2[EPV];
      rope_ld<T, EPV>(xr, x1);
      rope_ld<T, EPV>(xr + half, x2);
      rope_ld<T, EPV>(cs + tj, c);
      rope_ld<T, EPV>(sn + tj, s);
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        const float se = inverse ? -s[e] : s[e];
        const float a = V::rnd(__fmul_rn(x1[e], c[e])), bq = V::rnd(__fmul_rn(x2[e], se));
        const float d = V::rnd(__fmul_rn(x2[e], c[e])), f = V::rnd(__fmul_rn(x1[e], se));
        y1[e] = __fsub_rn(a, bq);
        y2[e] = __fadd_rn(d, f);
        if (inverse) {  // -0 -> +0, as the backward chain's adds onto zero-filled tensors give
          y1[e] = __fadd_rn(y1[e], 0.0f);
          y2[e] = __fadd_rn(y2[e], 0.0f);
        }
      }
      rope_st<T, EPV>(yr, y1);
      rope_st<T, EPV>(yr + half, y2);
    }
  }
}

template <typename T, int EPV>
static void rope_launch(void* y, const void* x, const void* cs, const void* sn, int64_t bh_n, int H,
                        int T_, int half, const RopeStrides& st, int inverse, cudaStream_t stream) {
  const int nvh = half / EPV, per_bh = T_ * nvh;
  const dim3 grid((unsigned)((per_bh + 255) / 256), (unsigned)(bh_n < 65535 ? bh_n : 65535));
  k_rope<T, EPV><<<grid, 256, 0, stream>>>((T*)y, (const T*)x, (const T*)cs, (const T*)sn, bh_n, H,
                                           per_bh, nvh, half, st, inverse);
}

// [lo, hi) byte range touched by a (B, H, T, 2*half) tensor with these element strides
static void rope_span(const void* p, const int64_t* s, int64_t B, int64_t H, int64_t T, int64_t half,
                      int es, uintptr_t* lo, uintptr_t* hi) {
  *lo = (uintptr_t)p;
  *hi = *lo + (uintptr_t)(((B - 1) * s[0] + (H - 1) * s[1] + (T - 1) * s[2] + 2 * half) * es);
}

}  // namespace edb

using namespace edb;

extern "C" {

int edb_rope(void* y, const void* x, const void* cos, const void* sin, int64_t B, int64_t H,
             int64_t T, int64_t half, const int64_t* x_strides, const int64_t* y_strides,
             int64_t table_stride_t, int inverse, int dtype, void* stream) {
  if (dtype != EDB_BF16 && dtype != EDB_F32) return set_error(EDB_E_UNSUPPORTED, "rope: dtype %d", dtype);
  if (half < 1 || half > kRopeMaxHalf)
    return set_error(EDB_E_UNSUPPORTED, "rope: head dim %lld (even, 2..%d)", (long long)(2 * half),
                     2 * kRopeMaxHalf);
  if (B < 0 || H < 0 || T < 0 || x_strides == nullptr || y_strides == nullptr)
    return set_error(EDB_E_INVALID, "rope: B=%lld H=%lld T=%lld, strides %p %p", (long long)B,
                     (long long)H, (long long)T, (const void*)x_strides, (const void*)y_strides);
  for (int k = 0; k < 3; ++k)
    if (x_strides[k] < 0 || y_strides[k] < 0) return set_error(EDB_E_INVALID, "rope: negative stride");
  if (table_stride_t < half) return set_error(EDB_E_INVALID, "rope: table stride %lld < half %lld",
                                              (long long)table_stride_t, (long long)half);
  if (B == 0 || H == 0 || T == 0) return EDB_OK;
  if (!y || !x || !cos || !sin) return set_error(EDB_E_INVALID, "rope: null pointer");
  if (T * half > (1LL << 30) || H > INT32_MAX)
    return set_error(EDB_E_UNSUPPORTED, "rope: T*half or H too large");
  const int es = dtype == EDB_BF16 ? 2 : 4, epv = 16 / es;
  uintptr_t xl, xh, yl, yh;
  rope_span(x, x_strides, B, H, T, half, es, &xl, &xh);
  rope_span(y, y_strides, B, H, T, half, es, &yl, &yh);
  if (yl < xh && xl < yh) return set_error(EDB_E_INVALID, "rope: y overlaps x");
  const RopeStrides st{x_strides[0], x_strides[1], x_strides[2],
                       y_strides[0], y_strides[1], y_strides[2], table_stride_t};
  bool vec = half % epv == 0 && table_stride_t % epv == 0 &&
             !(((uintptr_t)y | (uintptr_t)x | (uintptr_t)cos | (uintptr_t)sin) & 15);
  for (int k = 0; k < 3; ++k) vec = vec && x_strides[k] % epv == 0 && y_strides[k] % epv == 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t bh = B * H;
  if (dtype == EDB_BF16) {
    if (vec) rope_launch<__nv_bfloat16, 8>(y, x, cos, sin, bh, (int)H, (int)T, (int)half, st, inverse, s);
    else rope_launch<__nv_bfloat16, 1>(y, x, cos, sin, bh, (int)H, (int)T, (int)half, st, inverse, s);
  } else {
    if (vec) rope_launch<float, 4>(y, x, cos, sin, bh, (int)H, (int)T, (int)half, st, inverse, s);
    else rope_launch<float, 1>(y, x, cos, sin, bh, (int)H, (int)T, (int)half, st, inverse, s);
  }
  count_launch();
  return cuda_check(cudaGetLastError(), "k_rope launch");
}

}  // extern "C"
