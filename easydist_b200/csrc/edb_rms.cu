// RMSNorm and SwiGLU forward / backward for the sharded-op kernel dispatch of libedb.so.
//
// The Llama train step normalises with RMSNorm and gates its MLP with SwiGLU.  Traced, both are
// chains of elementwise ATen ops with fp32 intermediates of [tokens, H] / [tokens, ffn]; these kernels
// replace each chain by one HBM pass:
//   rms forward : rstd = rsqrt(mean(x^2) + eps) in fp32; y = T(T(x*rstd)*w) (RMS_CAST_THEN_SCALE, the
//                 hand-written Llama form) or T(x*rstd*w) (RMS_FUSED, aten._fused_rms_norm);
//                 2*R*H*sizeof(T) bytes
//   rms backward: n = x*rstd, g = dy*w; dx = T(add_in + rstd*(g - n*mean(g*n))) with one rounding;
//                 per-thread column partials of dw = sum(dy*n^) over all rows the thread sees, combined
//                 per CTA and finished by a second kernel in a fixed order (deterministic);
//                 3*R*H*sizeof(T) bytes (+ R*H with add_in)
//   swiglu      : out = T(T(silu(a))*b); dup = T(dy*T(silu(a))), dgate = silu_backward(T(dy*b), a),
//                 silu recomputed from a; 3 and 5 * n*sizeof(T) bytes
// Row layout: a row of H elements is nvec = H/EPV 16-byte vectors; a group of WPR warps owns a row and
// thread t of the group holds vectors t, t + 32*WPR, ... (NV per thread, predicated), so consecutive
// lanes read consecutive vectors.  Narrow rows take one warp per row (WPR = 1, rows in registers,
// the next row prefetched in the backward); wide rows take 2..16 warps per row.  The host picks
// (WPR, NV) from H.
#include <cuda_bf16.h>

#include "edb_internal.cuh"
#include "edb_vec.cuh"

namespace edb {

constexpr int kRmsMaxH = 16384;
constexpr int kRmsMaxCtasPerSm = 8;

template <typename T> using RmsT = VecT<T>;

__device__ __forceinline__ float rms_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// sum over the WPR warps of a row group; partials combined in warp order (deterministic).  Every
// thread of the CTA must call it (it synchronises when WPR > 1).
template <int WPR>
__device__ __forceinline__ float rms_group_sum(float v, float* red) {
  v = rms_warp_sum(v);
  if (WPR == 1) return v;
  const int warp = threadIdx.x >> 5, grp = warp / WPR;
  if ((threadIdx.x & 31) == 0) red[warp] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < WPR; ++k) s += red[grp * WPR + k];
  __syncthreads();
  return s;
}

// rows per CTA: 4 warps per CTA at least
template <int WPR> __host__ __device__ constexpr int rms_rows_per_cta() { return WPR >= 4 ? 1 : 4 / WPR; }
template <int WPR> __host__ __device__ constexpr int rms_threads() { return rms_rows_per_cta<WPR>() * WPR * 32; }

template <typename T, int WPR, int NV>
__global__ void __launch_bounds__(rms_threads<WPR>())
    k_rms_fwd(T* __restrict__ y, float* __restrict__ rstd, const T* __restrict__ x,
              const T* __restrict__ w, int64_t rows, int H, float eps, int fused) {
  constexpr int EPV = RmsT<T>::EPV;
  constexpr int RPC = rms_rows_per_cta<WPR>();
  __shared__ float red[RPC * WPR];
  const int t = threadIdx.x % (WPR * 32);
  const int64_t row = (int64_t)blockIdx.x * RPC + threadIdx.x / (WPR * 32);
  const bool live = row < rows;
  const int nvec = H / EPV;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (live ? row : 0) * H);
  float v[NV][EPV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = i * WPR * 32 + t;
    if (live && c < nvec) {
      RmsT<T>::unpack(xr[c], v[i]);
#pragma unroll
      for (int e = 0; e < EPV; ++e) s += v[i][e] * v[i][e];
    }
  }
  s = rms_group_sum<WPR>(s, red);
  if (!live) return;
  const float rs = rsqrtf(s / (float)H + eps);
  if (t == 0) rstd[row] = rs;
  uint4* yr = reinterpret_cast<uint4*>(y + row * H);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = i * WPR * 32 + t;
    if (c < nvec) {
      float wv[EPV], o[EPV];
      RmsT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(w) + c), wv);
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        const float n = v[i][e] * rs;
        o[e] = (fused ? n : RmsT<T>::rnd(n)) * wv[e];
      }
      yr[c] = RmsT<T>::pack(o);
    }
  }
}

// Persistent backward: grid-stride over row groups.  WPR == 1: the next row's x / dy vectors are
// requested before the current row is reduced (two rows in flight per warp); wider rows already have
// a whole row of loads in flight per CTA.  add_in is requested with x / dy when the registers allow.
template <typename T, int WPR, int NV>
__global__ void __launch_bounds__(rms_threads<WPR>(), (rms_threads<WPR>() <= 256 ? 2 : 1))
    k_rms_bwd(T* __restrict__ dx, float* __restrict__ part, const T* __restrict__ dy,
              const T* __restrict__ x, const float* __restrict__ rstd, const T* __restrict__ w,
              const T* __restrict__ add_in, int64_t rows, int H, int fused) {
  constexpr int EPV = RmsT<T>::EPV;
  constexpr int RPC = rms_rows_per_cta<WPR>();
  constexpr bool PF = (WPR == 1);
  constexpr bool PRE_ADD = (NV * 4 <= 16);
  __shared__ float red[RPC * WPR];
  extern __shared__ float rms_smem[];  // [RPC][H] when RPC > 1
  const int t = threadIdx.x % (WPR * 32), grp = threadIdx.x / (WPR * 32);
  const int nvec = H / EPV;
  const float inv_h = 1.0f / (float)H;
  float dwa[NV][EPV];
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int e = 0; e < EPV; ++e) dwa[i][e] = 0.f;
  const int64_t stride = (int64_t)gridDim.x * RPC;
  const int64_t first = (int64_t)blockIdx.x * RPC + grp;
  // all row groups of a CTA run the same number of iterations (group sums synchronise the CTA)
  const int64_t iters = rows > (int64_t)blockIdx.x * RPC
                            ? ((rows - (int64_t)blockIdx.x * RPC) + stride - 1) / stride : 0;
  uint4 xq[PF ? NV : 1], gq[PF ? NV : 1];
  float rs_n = 0.f;
  if (PF && first < rows) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = i * 32 + t;
      if (c < nvec) {
        xq[PF ? i : 0] = __ldg(reinterpret_cast<const uint4*>(x + first * H) + c);
        gq[PF ? i : 0] = __ldg(reinterpret_cast<const uint4*>(dy + first * H) + c);
      }
    }
    rs_n = rstd[first];
  }
  for (int64_t it = 0; it < iters; ++it) {
    const int64_t row = first + it * stride;
    const bool live = row < rows;
    uint4 xc[NV], gc[NV];
    float rs = 0.f;
    if (PF) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        xc[i] = xq[PF ? i : 0];
        gc[i] = gq[PF ? i : 0];
      }
      rs = rs_n;
      const int64_t nxt = row + stride;
      if (nxt < rows) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          const int c = i * 32 + t;
          if (c < nvec) {
            xq[PF ? i : 0] = __ldg(reinterpret_cast<const uint4*>(x + nxt * H) + c);
            gq[PF ? i : 0] = __ldg(reinterpret_cast<const uint4*>(dy + nxt * H) + c);
          }
        }
        rs_n = rstd[nxt];
      }
    } else if (live) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = i * WPR * 32 + t;
        if (c < nvec) {
          xc[i] = __ldg(reinterpret_cast<const uint4*>(x + row * H) + c);
          gc[i] = __ldg(reinterpret_cast<const uint4*>(dy + row * H) + c);
        }
      }
      rs = rstd[row];
    }
    uint4 ac[PRE_ADD ? NV : 1];
    if (PRE_ADD && live && add_in != nullptr) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = i * WPR * 32 + t;
        if (c < nvec) ac[PRE_ADD ? i : 0] = __ldg(reinterpret_cast<const uint4*>(add_in + row * H) + c);
      }
    }
    // s = sum(g*n) over the row; dw partials dy*n^ (n^ = T(n) in RMS_CAST_THEN_SCALE)
    float s = 0.f;
    if (live) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = i * WPR * 32 + t;
        if (c < nvec) {
          float xv[EPV], gv[EPV], wv[EPV];
          RmsT<T>::unpack(xc[i], xv);
          RmsT<T>::unpack(gc[i], gv);
          RmsT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(w) + c), wv);
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            const float n = xv[e] * rs;
            const float g = fused ? gv[e] * wv[e] : RmsT<T>::rnd(gv[e] * wv[e]);
            s += g * n;
            dwa[i][e] += gv[e] * (fused ? n : RmsT<T>::rnd(n));
          }
        }
      }
    }
    s = rms_group_sum<WPR>(s, red) * inv_h;
    if (!live) continue;
    uint4* dr = reinterpret_cast<uint4*>(dx + row * H);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = i * WPR * 32 + t;
      if (c < nvec) {
        float xv[EPV], gv[EPV], wv[EPV], o[EPV];
        RmsT<T>::unpack(xc[i], xv);
        RmsT<T>::unpack(gc[i], gv);
        RmsT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(w) + c), wv);
#pragma unroll
        for (int e = 0; e < EPV; ++e) {
          const float n = xv[e] * rs;
          const float g = fused ? gv[e] * wv[e] : RmsT<T>::rnd(gv[e] * wv[e]);
          o[e] = rs * (g - n * s);
        }
        if (add_in != nullptr) {
          float av[EPV];
          RmsT<T>::unpack(PRE_ADD ? ac[PRE_ADD ? i : 0]
                                  : __ldg(reinterpret_cast<const uint4*>(add_in + row * H) + c),
                          av);
#pragma unroll
          for (int e = 0; e < EPV; ++e) o[e] += av[e];
        }
        dr[c] = RmsT<T>::pack(o);
      }
    }
  }
  // one partial row of dw per CTA: row groups combined in group order
  if (part == nullptr) return;
  if constexpr (RPC == 1) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = i * WPR * 32 + t;
      if (c < nvec)
#pragma unroll
        for (int e = 0; e < EPV; ++e) part[(int64_t)blockIdx.x * H + c * EPV + e] = dwa[i][e];
    }
  } else {
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = i * WPR * 32 + t;
    if (c < nvec)
#pragma unroll
      for (int e = 0; e < EPV; ++e) rms_smem[grp * H + c * EPV + e] = dwa[i][e];
  }
  __syncthreads();
  for (int col = threadIdx.x; col < H; col += blockDim.x) {
    float a = 0.f;
#pragma unroll
    for (int k = 0; k < RPC; ++k) a += rms_smem[k * H + col];
    part[(int64_t)blockIdx.x * H + col] = a;
  }
  }
}

// dw[col] = T(sum over CTAs of part[cta][col]): 32 columns x 8 slices of CTAs per CTA, slices
// combined in a fixed order
template <typename T>
__global__ void __launch_bounds__(256)
    k_rms_bwd_finish(T* __restrict__ dw, const float* __restrict__ part, int n_part, int H) {
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + cx;
  float a = 0.f;
  if (col < H)
    for (int r = ry; r < n_part; r += 8) a += part[(int64_t)r * H + col];
  red[ry][cx] = a;
  __syncthreads();
  if (ry == 0 && col < H) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += red[k][cx];
    dw[col] = (T)s;
  }
}

// ---- host-side configuration --------------------------------------------------------------------

// (WPR, NV) for a row of nvec vectors: one warp per row up to 4 vectors per lane, then 2..16 warps
// with 4 vectors per lane (bf16 up to H = 16384, f32 up to 8192), f32 beyond with 16 warps x 8.
static bool rms_config(int64_t nvec, int* wpr, int* nv) {
  if (nvec <= 0) return false;
  if (nvec <= 32) { *wpr = 1; *nv = 1; return true; }
  if (nvec <= 64) { *wpr = 1; *nv = 2; return true; }
  if (nvec <= 128) { *wpr = 1; *nv = 4; return true; }
  for (int w = 2; w <= 16; w *= 2)
    if (nvec <= (int64_t)w * 32 * 4) { *wpr = w; *nv = 4; return true; }
  if (nvec <= 16 * 32 * 8) { *wpr = 16; *nv = 8; return true; }
  return false;
}

static int rms_epv(int dtype) { return dtype == EDB_BF16 ? 8 : 4; }

static bool rms_shape_ok(int64_t H, int dtype, int* wpr, int* nv) {
  if (dtype != EDB_BF16 && dtype != EDB_F32) return false;
  const int epv = rms_epv(dtype);
  return H > 0 && H <= kRmsMaxH && H % epv == 0 && rms_config(H / epv, wpr, nv);
}

// NV8: 8 for f32 (rows of more than 8192 elements); bf16 never selects it and passes 4
#define RMS_DISPATCH(WPRV, NVV, NV8, CALL)                                                      \
  do {                                                                                     \
    if (WPRV == 1 && NVV == 1) { constexpr int WPR = 1, NV = 1; CALL; }                    \
    else if (WPRV == 1 && NVV == 2) { constexpr int WPR = 1, NV = 2; CALL; }               \
    else if (WPRV == 1 && NVV == 4) { constexpr int WPR = 1, NV = 4; CALL; }               \
    else if (WPRV == 2) { constexpr int WPR = 2, NV = 4; CALL; }                           \
    else if (WPRV == 4) { constexpr int WPR = 4, NV = 4; CALL; }                           \
    else if (WPRV == 8) { constexpr int WPR = 8, NV = 4; CALL; }                           \
    else if (NVV == 4) { constexpr int WPR = 16, NV = 4; CALL; }                           \
    else { constexpr int WPR = 16, NV = NV8; CALL; }                                         \
  } while (0)

template <typename T, int WPR, int NV>
static void rms_fwd_launch(void* y, void* rstd, const void* x, const void* w, int64_t rows, int H,
                           float eps, int fused, cudaStream_t st) {
  constexpr int RPC = rms_rows_per_cta<WPR>();
  const int64_t grid = (rows + RPC - 1) / RPC;
  k_rms_fwd<T, WPR, NV><<<(unsigned)grid, rms_threads<WPR>(), 0, st>>>(
      (T*)y, (float*)rstd, (const T*)x, (const T*)w, rows, H, eps, fused);
}

// resident CTAs of the backward kernel per SM (occupancy query, capped); the grid and with it the
// dw summation order depend only on H, dtype and the device
template <typename T, int WPR, int NV>
static int rms_bwd_ctas_per_sm(int H) {
  auto kern = k_rms_bwd<T, WPR, NV>;
  constexpr int RPC = rms_rows_per_cta<WPR>();
  const int smem = RPC > 1 ? RPC * H * (int)sizeof(float) : 0;
  int n = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, rms_threads<WPR>(), smem) != cudaSuccess)
    n = 1;
  return n < 1 ? 1 : (n > kRmsMaxCtasPerSm ? kRmsMaxCtasPerSm : n);
}

template <typename T, int WPR, int NV>
static int rms_bwd_launch(void* dx, float* part, const void* dy, const void* x, const void* rstd,
                          const void* w, const void* add_in, int64_t rows, int H, int fused,
                          cudaStream_t st, int* grid_out) {
  constexpr int RPC = rms_rows_per_cta<WPR>();
  const int smem = RPC > 1 ? RPC * H * (int)sizeof(float) : 0;
  int64_t grid = (int64_t)rms_bwd_ctas_per_sm<T, WPR, NV>(H) * rt().sm_count;
  const int64_t row_ctas = (rows + RPC - 1) / RPC;
  if (grid > row_ctas) grid = row_ctas;
  k_rms_bwd<T, WPR, NV><<<(unsigned)grid, rms_threads<WPR>(), smem, st>>>(
      (T*)dx, part, (const T*)dy, (const T*)x, (const float*)rstd, (const T*)w, (const T*)add_in,
      rows, H, fused);
  *grid_out = (int)grid;
  return EDB_OK;
}

template <typename T, int WPR, int NV>
static size_t rms_bwd_ws_bytes(int H) {
  return (size_t)rms_bwd_ctas_per_sm<T, WPR, NV>(H) * rt().sm_count * (size_t)H * sizeof(float);
}

// ---- SwiGLU -------------------------------------------------------------------------------------

// The fp32 formulas of ATen's CUDA silu / silu_backward kernels (IEEE division, full-precision expf):
// results are bit-identical to the ATen chains.
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float silu_bwd_f(float dy, float x) {
  const float s = 1.0f / (1.0f + expf(-x));
  return dy * s * (1.0f + x * (1.0f - s));
}

template <typename T>
__device__ __forceinline__ void swiglu_fwd_elem(float a, float b, float& o) {
  o = RmsT<T>::rnd(silu_f(a)) * b;
}
template <typename T>
__device__ __forceinline__ void swiglu_bwd_elem(float g, float a, float b, float& da, float& db) {
  db = g * RmsT<T>::rnd(silu_f(a));
  da = silu_bwd_f(RmsT<T>::rnd(g * b), a);
}

// vec != 0: all pointers 16-byte aligned, vectors [0, n/EPV) then a scalar tail; else scalar
template <typename T>
__global__ void __launch_bounds__(256)
    k_swiglu_fwd(T* __restrict__ out, const T* __restrict__ a, const T* __restrict__ b, int64_t n,
                 int vec) {
  constexpr int EPV = RmsT<T>::EPV;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nth = (int64_t)gridDim.x * blockDim.x;
  int64_t done = 0;
  if (vec) {
    const int64_t nv = n / EPV;
    for (int64_t v = tid; v < nv; v += nth) {
      float av[EPV], bv[EPV], o[EPV];
      RmsT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(a) + v), av);
      RmsT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(b) + v), bv);
#pragma unroll
      for (int e = 0; e < EPV; ++e) swiglu_fwd_elem<T>(av[e], bv[e], o[e]);
      reinterpret_cast<uint4*>(out)[v] = RmsT<T>::pack(o);
    }
    done = nv * EPV;
  }
  for (int64_t i = done + tid; i < n; i += nth) {
    float o;
    swiglu_fwd_elem<T>(RmsT<T>::ld(a + i), RmsT<T>::ld(b + i), o);
    RmsT<T>::st(out + i, o);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
    k_swiglu_bwd(T* __restrict__ da, T* __restrict__ db, const T* __restrict__ dy,
                 const T* __restrict__ a, const T* __restrict__ b, int64_t n, int vec) {
  constexpr int EPV = RmsT<T>::EPV;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nth = (int64_t)gridDim.x * blockDim.x;
  int64_t done = 0;
  if (vec) {
    const int64_t nv = n / EPV;
    for (int64_t v = tid; v < nv; v += nth) {
      float gv[EPV], av[EPV], bv[EPV], oa[EPV], ob[EPV];
      RmsT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(dy) + v), gv);
      RmsT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(a) + v), av);
      RmsT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(b) + v), bv);
#pragma unroll
      for (int e = 0; e < EPV; ++e) swiglu_bwd_elem<T>(gv[e], av[e], bv[e], oa[e], ob[e]);
      reinterpret_cast<uint4*>(da)[v] = RmsT<T>::pack(oa);
      reinterpret_cast<uint4*>(db)[v] = RmsT<T>::pack(ob);
    }
    done = nv * EPV;
  }
  for (int64_t i = done + tid; i < n; i += nth) {
    float oa, ob;
    swiglu_bwd_elem<T>(RmsT<T>::ld(dy + i), RmsT<T>::ld(a + i), RmsT<T>::ld(b + i), oa, ob);
    RmsT<T>::st(da + i, oa);
    RmsT<T>::st(db + i, ob);
  }
}

// grid-stride launch: enough 256-thread CTAs to cover the work once, at most 8 per SM
static int swiglu_grid(int64_t work) {
  int64_t g = (work + 255) / 256;
  const int64_t cap = (int64_t)8 * rt().sm_count;
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}

}  // namespace edb

using namespace edb;

extern "C" {

int edb_rms_norm_fwd(void* y, void* rstd, const void* x, const void* w, int64_t rows, int64_t H,
                     float eps, int mode, int dtype, void* stream) {
  int wpr, nv;
  if (!rms_shape_ok(H, dtype, &wpr, &nv))
    return set_error(EDB_E_UNSUPPORTED, "rms_norm: H=%lld dtype %d not supported", (long long)H, dtype);
  if (mode != EDB_RMS_CAST_THEN_SCALE && mode != EDB_RMS_FUSED)
    return set_error(EDB_E_INVALID, "rms_norm: mode %d", mode);
  if (((uintptr_t)y | (uintptr_t)x | (uintptr_t)w) & 15)
    return set_error(EDB_E_UNSUPPORTED, "rms_norm: pointers must be 16-byte aligned");
  if (rows <= 0) return EDB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int fused = mode == EDB_RMS_FUSED;
  if (dtype == EDB_BF16)
    RMS_DISPATCH(wpr, nv, 4, (rms_fwd_launch<__nv_bfloat16, WPR, NV>(y, rstd, x, w, rows, (int)H, eps, fused, st)));
  else
    RMS_DISPATCH(wpr, nv, 8, (rms_fwd_launch<float, WPR, NV>(y, rstd, x, w, rows, (int)H, eps, fused, st)));
  count_launch();
  return cuda_check(cudaGetLastError(), "k_rms_fwd launch");
}

// enough for either dtype at this H
int edb_rms_norm_bwd_workspace(int64_t H, size_t* bytes_out) {
  int wpr, nv;
  size_t bytes = 0, b = 0;
  if (rms_shape_ok(H, EDB_BF16, &wpr, &nv)) {
    RMS_DISPATCH(wpr, nv, 4, (b = rms_bwd_ws_bytes<__nv_bfloat16, WPR, NV>((int)H)));
    bytes = b;
  }
  if (rms_shape_ok(H, EDB_F32, &wpr, &nv)) {
    RMS_DISPATCH(wpr, nv, 8, (b = rms_bwd_ws_bytes<float, WPR, NV>((int)H)));
    if (b > bytes) bytes = b;
  }
  if (bytes == 0)
    return set_error(EDB_E_UNSUPPORTED, "rms_norm_bwd: H=%lld not supported", (long long)H);
  *bytes_out = bytes;
  return EDB_OK;
}

int edb_rms_norm_bwd(void* dx, void* dw, const void* dy, const void* x, const void* rstd,
                     const void* w, const void* add_in, void* workspace, int64_t rows, int64_t H,
                     int mode, int dtype, void* stream) {
  int wpr, nv;
  if (!rms_shape_ok(H, dtype, &wpr, &nv))
    return set_error(EDB_E_UNSUPPORTED, "rms_norm_bwd: H=%lld dtype %d not supported", (long long)H,
                     dtype);
  if (mode != EDB_RMS_CAST_THEN_SCALE && mode != EDB_RMS_FUSED)
    return set_error(EDB_E_INVALID, "rms_norm_bwd: mode %d", mode);
  if (((uintptr_t)dx | (uintptr_t)dy | (uintptr_t)x | (uintptr_t)w | (uintptr_t)add_in |
       (uintptr_t)workspace) & 15)
    return set_error(EDB_E_UNSUPPORTED, "rms_norm_bwd: pointers must be 16-byte aligned");
  if (rows <= 0) return EDB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int fused = mode == EDB_RMS_FUSED;
  float* part = dw != nullptr ? static_cast<float*>(workspace) : nullptr;
  int grid = 0, rc = EDB_OK;
  if (dtype == EDB_BF16)
    RMS_DISPATCH(wpr, nv, 4, (rc = rms_bwd_launch<__nv_bfloat16, WPR, NV>(dx, part, dy, x, rstd, w, add_in, rows, (int)H, fused, st, &grid)));
  else
    RMS_DISPATCH(wpr, nv, 8, (rc = rms_bwd_launch<float, WPR, NV>(dx, part, dy, x, rstd, w, add_in, rows, (int)H, fused, st, &grid)));
  if (rc) return rc;
  count_launch();
  if (dw != nullptr) {
    const int fin = (int)((H + 31) / 32);
    if (dtype == EDB_BF16)
      k_rms_bwd_finish<__nv_bfloat16><<<fin, 256, 0, st>>>((__nv_bfloat16*)dw, part, grid, (int)H);
    else
      k_rms_bwd_finish<float><<<fin, 256, 0, st>>>((float*)dw, part, grid, (int)H);
    count_launch();
  }
  return cuda_check(cudaGetLastError(), "k_rms_bwd launch");
}

int edb_swiglu_fwd(void* out, const void* gate, const void* up, int64_t n, int dtype, void* stream) {
  if (dtype != EDB_BF16 && dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "swiglu: dtype %d", dtype);
  if (n <= 0) return EDB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int vec = !(((uintptr_t)out | (uintptr_t)gate | (uintptr_t)up) & 15);
  const int64_t work = vec ? n / rms_epv(dtype) + 1 : n;
  if (dtype == EDB_BF16)
    k_swiglu_fwd<__nv_bfloat16><<<swiglu_grid(work), 256, 0, st>>>(
        (__nv_bfloat16*)out, (const __nv_bfloat16*)gate, (const __nv_bfloat16*)up, n, vec);
  else
    k_swiglu_fwd<float><<<swiglu_grid(work), 256, 0, st>>>((float*)out, (const float*)gate,
                                                           (const float*)up, n, vec);
  count_launch();
  return cuda_check(cudaGetLastError(), "k_swiglu_fwd launch");
}

int edb_swiglu_bwd(void* dgate, void* dup, const void* dy, const void* gate, const void* up,
                   int64_t n, int dtype, void* stream) {
  if (dtype != EDB_BF16 && dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "swiglu_bwd: dtype %d", dtype);
  if (n <= 0) return EDB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int vec = !(((uintptr_t)dgate | (uintptr_t)dup | (uintptr_t)dy | (uintptr_t)gate |
                     (uintptr_t)up) & 15);
  const int64_t work = vec ? n / rms_epv(dtype) + 1 : n;
  if (dtype == EDB_BF16)
    k_swiglu_bwd<__nv_bfloat16><<<swiglu_grid(work), 256, 0, st>>>(
        (__nv_bfloat16*)dgate, (__nv_bfloat16*)dup, (const __nv_bfloat16*)dy,
        (const __nv_bfloat16*)gate, (const __nv_bfloat16*)up, n, vec);
  else
    k_swiglu_bwd<float><<<swiglu_grid(work), 256, 0, st>>>((float*)dgate, (float*)dup,
                                                           (const float*)dy, (const float*)gate,
                                                           (const float*)up, n, vec);
  count_launch();
  return cuda_check(cudaGetLastError(), "k_swiglu_bwd launch");
}

}  // extern "C"
