// LayerNorm forward / backward for the sharded-op kernel dispatch of libedb.so.
//
// aten.native_layer_norm(_backward) is a large non-GEMM item of the GPT-2 train step: 49 backward
// calls per step on [4096,1024] bf16 activations, each far above its HBM streaming floor.
// These kernels are pure HBM streaming with warp-level reductions:
//   forward : one warp per row, the row lives in registers (16-byte vector loads), two-pass
//             mean/variance by shuffles, y = (x-mean)*rstd*w + b; 2*R*H*sizeof(T) bytes moved
//   backward: persistent grid (one CTA per SM, 4 warps), one warp per row:
//             dx = rstd*(g - mean(g) - xhat*mean(g*xhat)), g = dy*w; per-lane column partials of
//             dw = sum(dy*xhat), db = sum(dy) stay in registers over all rows of the warp, are
//             combined per CTA in shared memory and finished by a second tiny kernel in a fixed
//             order (deterministic); 3*R*H*sizeof(T) bytes moved
// Semantics: aten.native_layer_norm / native_layer_norm_backward over the last dimension
// (mean/rstd are fp32, shape [..., 1]), the ops the reference's traced graph contains
// (SURVEY.md App. B: native_layer_norm(+bwd) 8+8 per step in config 1).
#include <cuda_bf16.h>

#include "edb_internal.cuh"
#include "edb_vec.cuh"

namespace edb {

constexpr int kLnWarps = 4;
constexpr int kLnMaxVec = 16;  // 16-byte vectors per lane: H <= 32*16*EPV

template <typename T> using LnT = VecT<T>;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// vector v of lane l covers elements [(v*32 + l)*EPV, +EPV): consecutive lanes read consecutive
// 16-byte vectors (fully coalesced 512-byte warp requests)
template <typename T, int NV>
__global__ void __launch_bounds__(kLnWarps * 32)
    k_ln_fwd(T* __restrict__ y, float* __restrict__ mean, float* __restrict__ rstd,
             const T* __restrict__ x, const T* __restrict__ w, const T* __restrict__ b, int64_t rows,
             int H, float eps) {
  constexpr int EPV = LnT<T>::EPV;
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kLnWarps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * H);
  float v[NV][EPV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const uint4 raw = xr[i * 32 + lane];
    LnT<T>::unpack(raw, v[i]);
#pragma unroll
    for (int e = 0; e < EPV; ++e) s += v[i][e];
  }
  const float mu = warp_sum(s) / (float)H;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int e = 0; e < EPV; ++e) {
      const float d = v[i][e] - mu;
      q += d * d;
    }
  const float rs = rsqrtf(warp_sum(q) / (float)H + eps);
  if (lane == 0) {
    mean[row] = mu;
    rstd[row] = rs;
  }
  uint4* yr = reinterpret_cast<uint4*>(y + row * H);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    float wv[EPV], bv[EPV], o[EPV];
    LnT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(w) + i * 32 + lane), wv);
    if (b != nullptr) LnT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(b) + i * 32 + lane), bv);
#pragma unroll
    for (int e = 0; e < EPV; ++e) {
      o[e] = (v[i][e] - mu) * rs * wv[e];
      if (b != nullptr) o[e] += bv[e];
    }
    yr[i * 32 + lane] = LnT<T>::pack(o);
  }
}

template <typename T, int NV>
__global__ void __launch_bounds__(kLnWarps * 32, (NV <= 4 ? 2 : 1))
    k_ln_bwd(T* __restrict__ dx, float* __restrict__ part, const T* __restrict__ dy,
             const T* __restrict__ x, const float* __restrict__ mean,
             const float* __restrict__ rstd, const T* __restrict__ w, int64_t rows, int H,
             const T* __restrict__ add_in) {
  constexpr int EPV = LnT<T>::EPV;
  extern __shared__ float ln_smem[];  // [kLnWarps][2][H]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float wv[NV][EPV], dwa[NV][EPV], dba[NV][EPV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    LnT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(w) + i * 32 + lane), wv[i]);
#pragma unroll
    for (int e = 0; e < EPV; ++e) dwa[i][e] = dba[i][e] = 0.f;
  }
  const float inv_h = 1.0f / (float)H;
  const int64_t stride = (int64_t)gridDim.x * kLnWarps;
  int64_t row = (int64_t)blockIdx.x * kLnWarps + warp;
  // NV <= 4 (H <= 1024 bf16): the next row's x / dy vectors are requested before the current row
  // is reduced, so every warp keeps two rows (4 * NV 16-byte loads per lane) in flight; wider rows
  // already carry that many loads per row and would spill with the extra buffers
  constexpr bool PF = (NV <= 4);
  uint4 xq[PF ? NV : 1], gq[PF ? NV : 1];
  float mu_n = 0.f, rs_n = 0.f;
  if (PF && row < rows) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      xq[PF ? i : 0] = __ldg(reinterpret_cast<const uint4*>(x + row * H) + i * 32 + lane);
      gq[PF ? i : 0] = __ldg(reinterpret_cast<const uint4*>(dy + row * H) + i * 32 + lane);
    }
    mu_n = mean[row];
    rs_n = rstd[row];
  }
  for (; row < rows; row += stride) {
    uint4 xc[NV], gc[NV];
    float mu, rs;
    if (PF) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        xc[i] = xq[PF ? i : 0];
        gc[i] = gq[PF ? i : 0];
      }
      mu = mu_n;
      rs = rs_n;
      const int64_t nxt = row + stride;
      if (nxt < rows) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          xq[PF ? i : 0] = __ldg(reinterpret_cast<const uint4*>(x + nxt * H) + i * 32 + lane);
          gq[PF ? i : 0] = __ldg(reinterpret_cast<const uint4*>(dy + nxt * H) + i * 32 + lane);
        }
        mu_n = mean[nxt];
        rs_n = rstd[nxt];
      }
    } else {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        xc[i] = __ldg(reinterpret_cast<const uint4*>(x + row * H) + i * 32 + lane);
        gc[i] = __ldg(reinterpret_cast<const uint4*>(dy + row * H) + i * 32 + lane);
      }
      mu = mean[row];
      rs = rstd[row];
    }
    // fused gradient accumulation: dx = T(T(dx_ln) + add_in[row]) — the aten.add.Tensor that joins the
    // LayerNorm branch with the residual branch in the backward pass (same two roundings as ATen)
    uint4 ac[NV];
    if (add_in != nullptr) {
#pragma unroll
      for (int i = 0; i < NV; ++i)
        ac[i] = __ldg(reinterpret_cast<const uint4*>(add_in + row * H) + i * 32 + lane);
    }
    float xh[NV][EPV], g[NV][EPV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float xv[EPV], gv[EPV];
      LnT<T>::unpack(xc[i], xv);
      LnT<T>::unpack(gc[i], gv);
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        xh[i][e] = (xv[e] - mu) * rs;
        g[i][e] = gv[e] * wv[i][e];
        s1 += g[i][e];
        s2 += g[i][e] * xh[i][e];
        dwa[i][e] += gv[e] * xh[i][e];
        dba[i][e] += gv[e];
      }
    }
    s1 = warp_sum(s1) * inv_h;
    s2 = warp_sum(s2) * inv_h;
    uint4* dr = reinterpret_cast<uint4*>(dx + row * H);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float o[EPV];
#pragma unroll
      for (int e = 0; e < EPV; ++e) o[e] = rs * (g[i][e] - s1 - xh[i][e] * s2);
      if (add_in != nullptr) {
        float r1[EPV], av[EPV];
        LnT<T>::unpack(LnT<T>::pack(o), r1);  // round to T first, like the separate kernels do
        LnT<T>::unpack(ac[i], av);
#pragma unroll
        // __fadd_rn: for T = float the rounding to T is a no-op, and a plain + would be contracted
        // with the product above into one FMA (one rounding instead of ATen's two)
        for (int e = 0; e < EPV; ++e) o[e] = __fadd_rn(r1[e], av[e]);
      }
      dr[i * 32 + lane] = LnT<T>::pack(o);
    }
  }
  // CTA-level combine of the warps' column partials (fixed warp order), then one partial row per CTA
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int e = 0; e < EPV; ++e) {
      const int col = (i * 32 + lane) * EPV + e;
      ln_smem[(warp * 2 + 0) * H + col] = dwa[i][e];
      ln_smem[(warp * 2 + 1) * H + col] = dba[i][e];
    }
  __syncthreads();
  for (int col = threadIdx.x; col < H; col += blockDim.x) {
    float a = 0.f, c = 0.f;
#pragma unroll
    for (int k = 0; k < kLnWarps; ++k) {
      a += ln_smem[(k * 2 + 0) * H + col];
      c += ln_smem[(k * 2 + 1) * H + col];
    }
    part[((int64_t)blockIdx.x * 2 + 0) * H + col] = a;
    part[((int64_t)blockIdx.x * 2 + 1) * H + col] = c;
  }
}

// dw[col] = sum over CTAs of part[cta][0][col]; db likewise.  32 columns x 8 row slices per CTA.
template <typename T>
__global__ void __launch_bounds__(256)
    k_ln_bwd_finish(T* __restrict__ dw, T* __restrict__ db, const float* __restrict__ part,
                    int n_part, int H) {
  __shared__ float red[2][8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + cx;
  float a = 0.f, c = 0.f;
  if (col < H)
    for (int r = ry; r < n_part; r += 8) {
      a += part[((int64_t)r * 2 + 0) * H + col];
      c += part[((int64_t)r * 2 + 1) * H + col];
    }
  red[0][ry][cx] = a;
  red[1][ry][cx] = c;
  __syncthreads();
  if (ry == 0 && col < H) {
    float sa = 0.f, sc = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      sa += red[0][k][cx];
      sc += red[1][k][cx];
    }
    if (dw) dw[col] = (T)sa;
    if (db) db[col] = (T)sc;
  }
}

// Column sums out[c] = sum_r x[r, c] (bias gradients: aten.sum.dim_IntList(dy, [0], True), 96 per
// GPT-2-medium step).  Grid = column stripes (32 lanes x EPV columns) x row splits; every lane owns
// EPV consecutive columns (16-byte loads, coalesced along the row); 8 warps interleave the rows of a
// split and each keeps 8 independent row loads in flight (32 KB per CTA), so that a [4096,1024]
// bf16 operand (8 MB) is entirely in flight at once.  Partials are combined in a fixed order.
constexpr int kCsWarps = 8;
constexpr int kCsUnroll = 8;
constexpr int kCsMaxSplits = 128;

template <typename T>
__global__ void __launch_bounds__(kCsWarps * 32)
    k_colsum(float* __restrict__ part, const T* __restrict__ x, int64_t rows, int64_t cols,
             int64_t ld, int rows_per_split) {
  constexpr int EPV = LnT<T>::EPV;
  __shared__ float red[kCsWarps][32 * EPV];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t col = ((int64_t)blockIdx.x * 32 + lane) * EPV;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_split;
  const int64_t r1 = r0 + rows_per_split < rows ? r0 + rows_per_split : rows;
  float acc[EPV];
#pragma unroll
  for (int e = 0; e < EPV; ++e) acc[e] = 0.f;
  if (col < cols) {
    int64_t r = r0 + warp;
    for (; r + (kCsUnroll - 1) * kCsWarps < r1; r += kCsUnroll * kCsWarps) {
      uint4 raw[kCsUnroll];
#pragma unroll
      for (int u = 0; u < kCsUnroll; ++u)
        raw[u] = __ldg(reinterpret_cast<const uint4*>(x + (r + u * kCsWarps) * ld + col));
#pragma unroll
      for (int u = 0; u < kCsUnroll; ++u) {
        float f[EPV];
        LnT<T>::unpack(raw[u], f);
#pragma unroll
        for (int e = 0; e < EPV; ++e) acc[e] += f[e];
      }
    }
    for (; r < r1; r += kCsWarps) {
      float f[EPV];
      LnT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(x + r * ld + col)), f);
#pragma unroll
      for (int e = 0; e < EPV; ++e) acc[e] += f[e];
    }
  }
#pragma unroll
  for (int e = 0; e < EPV; ++e) red[warp][lane * EPV + e] = acc[e];
  __syncthreads();
  for (int i = threadIdx.x; i < 32 * EPV; i += blockDim.x) {
    const int64_t c = (int64_t)blockIdx.x * 32 * EPV + i;
    if (c < cols) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < kCsWarps; ++k) s += red[k][i];
      part[(int64_t)blockIdx.y * cols + c] = s;
    }
  }
}

// out[c] = sum over splits of part[k][c]: 32 columns x 8 slices of k per CTA (independent loads),
// slices combined in a fixed order.
template <typename T>
__global__ void __launch_bounds__(256)
    k_colsum_finish(T* __restrict__ out, const float* __restrict__ part, int n_part, int64_t cols) {
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, ky = threadIdx.x >> 5;
  const int64_t c = (int64_t)blockIdx.x * 32 + cx;
  float s = 0.f;
  if (c < cols) {
#pragma unroll 4
    for (int k = ky; k < n_part; k += 8) s += part[(int64_t)k * cols + c];
  }
  red[ky][cx] = s;
  __syncthreads();
  if (ky == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][cx];
    out[c] = (T)t;
  }
}

template <typename T> static bool ln_shape_ok(int64_t H) {
  const int per = 32 * LnT<T>::EPV;
  return H > 0 && H % per == 0 && H / per <= kLnMaxVec && H <= 2048;
}

template <typename T, int NV>
static void ln_fwd_launch(void* y, void* mean, void* rstd, const void* x, const void* w,
                          const void* b, int64_t rows, int H, float eps, cudaStream_t st) {
  const int grid = (int)((rows + kLnWarps - 1) / kLnWarps);
  k_ln_fwd<T, NV><<<grid, kLnWarps * 32, 0, st>>>((T*)y, (float*)mean, (float*)rstd, (const T*)x,
                                                  (const T*)w, (const T*)b, rows, H, eps);
}

template <typename T, int NV>
static int ln_bwd_launch(void* dx, float* part, const void* dy, const void* x, const void* mean,
                         const void* rstd, const void* w, int64_t rows, int H, int grid,
                         cudaStream_t st, const void* add_in) {
  auto kern = k_ln_bwd<T, NV>;
  const int smem = kLnWarps * 2 * H * (int)sizeof(float);
  static bool configured = false;
  if (!configured && smem > 48 * 1024) {
    EDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    configured = true;
  }
  kern<<<grid, kLnWarps * 32, smem, st>>>((T*)dx, part, (const T*)dy, (const T*)x,
                                          (const float*)mean, (const float*)rstd, (const T*)w, rows,
                                          H, (const T*)add_in);
  return EDB_OK;
}

#define LN_DISPATCH_NV(NVAR, CALL)                                   \
  switch (NVAR) {                                                    \
    case 1: { constexpr int NV = 1; CALL; } break;                   \
    case 2: { constexpr int NV = 2; CALL; } break;                   \
    case 3: { constexpr int NV = 3; CALL; } break;                   \
    case 4: { constexpr int NV = 4; CALL; } break;                   \
    case 6: { constexpr int NV = 6; CALL; } break;                   \
    case 8: { constexpr int NV = 8; CALL; } break;                   \
    default: return set_error(EDB_E_UNSUPPORTED, "layer_norm: H=%lld not supported", (long long)H); \
  }

}  // namespace edb

using namespace edb;

extern "C" {

int edb_layer_norm_bwd_workspace(int64_t H, size_t* bytes_out) {
  int sms = rt().sm_count;
  *bytes_out = (size_t)(2 * sms) * 2 * (size_t)H * sizeof(float);  // one partial pair per CTA, 2 CTAs/SM
  return EDB_OK;
}

int edb_colsum_workspace(int64_t cols, size_t* bytes_out) {
  *bytes_out = (size_t)kCsMaxSplits * (size_t)cols * sizeof(float);
  return EDB_OK;
}

int edb_colsum(void* out, const void* x, void* workspace, int64_t rows, int64_t cols, int64_t ld,
               int dtype, void* stream) {
  if (rows <= 0 || cols <= 0) return set_error(EDB_E_UNSUPPORTED, "edb_colsum: empty input");
  if (dtype != EDB_BF16 && dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "edb_colsum: dtype %d", dtype);
  const int epv = dtype == EDB_BF16 ? 8 : 4;
  if ((cols % epv) || (ld % epv) || (((uintptr_t)x | (uintptr_t)workspace) & 15))
    return set_error(EDB_E_UNSUPPORTED, "edb_colsum: cols/ld must be multiples of %d, 16-byte aligned",
                     epv);
  cudaStream_t st = (cudaStream_t)stream;
  const int stripes = (int)((cols + 32 * epv - 1) / (32 * epv));
  // about 4 CTAs per SM in total, but at least one full unrolled pass (64 rows) per split
  int splits = (4 * rt().sm_count + stripes - 1) / stripes;
  if (splits > kCsMaxSplits) splits = kCsMaxSplits;
  const int64_t min_rows = kCsWarps * kCsUnroll;
  if (splits > rows / min_rows) splits = (int)(rows / min_rows > 0 ? rows / min_rows : 1);
  if (splits < 1) splits = 1;
  const int rps = (int)((rows + splits - 1) / splits);
  splits = (int)((rows + rps - 1) / rps);
  float* part = static_cast<float*>(workspace);
  dim3 grid(stripes, splits);
  const int fin = (int)((cols + 31) / 32);
  if (dtype == EDB_BF16) {
    k_colsum<__nv_bfloat16><<<grid, kCsWarps * 32, 0, st>>>(part, (const __nv_bfloat16*)x, rows, cols,
                                                           ld, rps);
    k_colsum_finish<__nv_bfloat16><<<fin, 256, 0, st>>>((__nv_bfloat16*)out, part, splits, cols);
  } else {
    k_colsum<float><<<grid, kCsWarps * 32, 0, st>>>(part, (const float*)x, rows, cols, ld, rps);
    k_colsum_finish<float><<<fin, 256, 0, st>>>((float*)out, part, splits, cols);
  }
  count_launch();
  count_launch();
  return cuda_check(cudaGetLastError(), "k_colsum launch");
}

int edb_layer_norm_fwd(void* y, void* mean, void* rstd, const void* x, const void* w, const void* b,
                       int64_t rows, int64_t H, float eps, int dtype, void* stream) {
  if (rows <= 0) return EDB_OK;
  if (((uintptr_t)y | (uintptr_t)x | (uintptr_t)w | (uintptr_t)b) & 15)
    return set_error(EDB_E_UNSUPPORTED, "layer_norm: pointers must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == EDB_BF16) {
    if (!ln_shape_ok<__nv_bfloat16>(H))
      return set_error(EDB_E_UNSUPPORTED, "layer_norm: H=%lld not supported", (long long)H);
    const int nv = (int)(H / 256);
    LN_DISPATCH_NV(nv, (ln_fwd_launch<__nv_bfloat16, NV>(y, mean, rstd, x, w, b, rows, (int)H, eps, st)));
  } else if (dtype == EDB_F32) {
    if (!ln_shape_ok<float>(H))
      return set_error(EDB_E_UNSUPPORTED, "layer_norm: H=%lld not supported", (long long)H);
    const int nv = (int)(H / 128);
    LN_DISPATCH_NV(nv, (ln_fwd_launch<float, NV>(y, mean, rstd, x, w, b, rows, (int)H, eps, st)));
  } else {
    return set_error(EDB_E_UNSUPPORTED, "layer_norm: dtype %d", dtype);
  }
  count_launch();
  return cuda_check(cudaGetLastError(), "k_ln_fwd launch");
}

int edb_layer_norm_bwd(void* dx, void* dw, void* db, const void* dy, const void* x, const void* mean,
                       const void* rstd, const void* w, void* workspace, int64_t rows, int64_t H,
                       int dtype, void* stream) {
  return edb_layer_norm_bwd_add(dx, dw, db, dy, x, mean, rstd, w, nullptr, workspace, rows, H, dtype,
                                stream);
}

int edb_layer_norm_bwd_add(void* dx, void* dw, void* db, const void* dy, const void* x,
                           const void* mean, const void* rstd, const void* w, const void* add_in,
                           void* workspace, int64_t rows, int64_t H, int dtype, void* stream) {
  if (rows <= 0) return EDB_OK;
  if ((uintptr_t)add_in & 15)
    return set_error(EDB_E_UNSUPPORTED, "layer_norm_bwd: pointers must be 16-byte aligned");
  if (((uintptr_t)dx | (uintptr_t)dy | (uintptr_t)x | (uintptr_t)w | (uintptr_t)workspace) & 15)
    return set_error(EDB_E_UNSUPPORTED, "layer_norm_bwd: pointers must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  int grid = 2 * rt().sm_count;
  const int64_t row_ctas = (rows + kLnWarps - 1) / kLnWarps;
  if (grid > row_ctas) grid = (int)row_ctas;
  float* part = static_cast<float*>(workspace);
  int rc = EDB_OK;
  if (dtype == EDB_BF16) {
    if (!ln_shape_ok<__nv_bfloat16>(H))
      return set_error(EDB_E_UNSUPPORTED, "layer_norm_bwd: H=%lld not supported", (long long)H);
    const int nv = (int)(H / 256);
    LN_DISPATCH_NV(nv, (rc = ln_bwd_launch<__nv_bfloat16, NV>(dx, part, dy, x, mean, rstd, w, rows, (int)H, grid, st, add_in)));
    if (rc) return rc;
    k_ln_bwd_finish<__nv_bfloat16><<<(int)((H + 31) / 32), 256, 0, st>>>(
        (__nv_bfloat16*)dw, (__nv_bfloat16*)db, part, grid, (int)H);
  } else if (dtype == EDB_F32) {
    if (!ln_shape_ok<float>(H))
      return set_error(EDB_E_UNSUPPORTED, "layer_norm_bwd: H=%lld not supported", (long long)H);
    const int nv = (int)(H / 128);
    LN_DISPATCH_NV(nv, (rc = ln_bwd_launch<float, NV>(dx, part, dy, x, mean, rstd, w, rows, (int)H, grid, st, add_in)));
    if (rc) return rc;
    k_ln_bwd_finish<float><<<(int)((H + 31) / 32), 256, 0, st>>>((float*)dw, (float*)db, part, grid,
                                                                 (int)H);
  } else {
    return set_error(EDB_E_UNSUPPORTED, "layer_norm_bwd: dtype %d", dtype);
  }
  count_launch();
  count_launch();
  return cuda_check(cudaGetLastError(), "k_ln_bwd launch");
}

}  // extern "C"
