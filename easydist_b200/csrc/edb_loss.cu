// Cross-entropy (log-softmax + NLL) forward / backward for the sharded-op kernel dispatch.
//
// The traced train step of a language model ends in
//   mm (LM head) -> _to_copy(fp32) -> _log_softmax -> nll_loss_forward
// and its backward starts with
//   nll_loss_backward -> _log_softmax_backward_data -> _to_copy(bf16) -> mm x2
// (the ops the reference's graphs carry for its GPT example too: benchmark/torch/model/gpt.py +
// F.cross_entropy in examples/torch/gpt_train.py:37-43).  With a 50257-word vocabulary and 4096
// rows that chain moves ~8 GB through HBM per step in ATen (an fp32 copy of the logits, an fp32
// log-softmax, an fp32 gradient, a bf16 copy of it, plus two padded re-copies for the TMA
// alignment of the following GEMMs).
// Here the logits are read once in their storage dtype for the forward (online max / sum-exp per
// row, fp32 accumulation) and once for the backward, which writes the gradient straight into a
// TMA-legal (row stride % 8 == 0) bf16 buffer that the two LM-head GEMMs consume without staging:
// 3 * R * V * sizeof(T) bytes in total.
//
// Semantics: aten._log_softmax(dim=-1) + aten.nll_loss_forward(weight=None, reduction mean|sum,
// ignore_index) and their backward ops; loss / total_weight are fp32 scalars, reduction over rows in
// a fixed order (deterministic, same bits on every run).
#include <cuda_bf16.h>

#include "edb_internal.cuh"
#include "edb_vec.cuh"

namespace edb {

constexpr int kCeThreads = 256;
constexpr float kLog2e = 1.4426950408889634f;

template <typename T> using CeT = VecT<T>;

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// running (max, sum of exp(x - max)) pair; `m` is kept in the log2 domain (x * log2e)
struct MaxSum {
  float m, s;
};
__device__ __forceinline__ void ms_add_vec(MaxSum& a, const float* f, int n) {
  float vm = f[0];
#pragma unroll
  for (int e = 1; e < 8; ++e)
    if (e < n) vm = fmaxf(vm, f[e]);
  vm *= kLog2e;
  if (vm > a.m) {
    a.s *= fast_exp2(a.m - vm);  // a.m == -inf: s is 0 and stays 0 (ex2(-inf) = 0)
    a.m = vm;
  }
  if (a.m == -INFINITY) return;  // all entries -inf so far
#pragma unroll
  for (int e = 0; e < 8; ++e)
    if (e < n) a.s += fast_exp2(fmaf(f[e], kLog2e, -a.m));
}
__device__ __forceinline__ MaxSum ms_merge(const MaxSum& a, const MaxSum& b) {
  MaxSum o;
  o.m = fmaxf(a.m, b.m);
  if (o.m == -INFINITY) {
    o.s = 0.f;
    return o;
  }
  o.s = a.s * fast_exp2(a.m - o.m) + b.s * fast_exp2(b.m - o.m);
  return o;
}

// One CTA per row.  VEC = true: rows are 16-byte aligned (ld % EPV == 0, aligned base).
template <typename T, bool VEC>
__global__ void __launch_bounds__(kCeThreads)
    k_ce_fwd(float* __restrict__ lse, float* __restrict__ row_loss, const T* __restrict__ x,
             int64_t ld, const int64_t* __restrict__ target, int64_t vocab, int64_t ignore_index) {
  constexpr int EPV = CeT<T>::EPV;
  const int64_t row = blockIdx.x;
  const T* xr = x + row * ld;
  MaxSum acc = {-INFINITY, 0.f};
  if (VEC) {
    const int64_t nvec = vocab / EPV;
    const uint4* xv = reinterpret_cast<const uint4*>(xr);
    int64_t i = threadIdx.x;
    for (; i + 3 * kCeThreads < nvec; i += 4 * kCeThreads) {
      uint4 raw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) raw[u] = __ldg(xv + i + u * kCeThreads);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float f[8];
        CeT<T>::unpack(raw[u], f);
        ms_add_vec(acc, f, EPV);
      }
    }
    for (; i < nvec; i += kCeThreads) {
      float f[8];
      CeT<T>::unpack(__ldg(xv + i), f);
      ms_add_vec(acc, f, EPV);
    }
    for (int64_t j = nvec * EPV + threadIdx.x; j < vocab; j += kCeThreads) {
      float f[8];
      f[0] = CeT<T>::ld(xr + j);
      ms_add_vec(acc, f, 1);
    }
  } else {
    for (int64_t j = threadIdx.x; j < vocab; j += kCeThreads) {
      float f[8];
      f[0] = CeT<T>::ld(xr + j);
      ms_add_vec(acc, f, 1);
    }
  }
  // CTA reduction in a fixed order: lanes by xor-shuffle, then warps 0..7 sequentially
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MaxSum b;
    b.m = __shfl_xor_sync(0xffffffffu, acc.m, o);
    b.s = __shfl_xor_sync(0xffffffffu, acc.s, o);
    acc = ms_merge(acc, b);
  }
  __shared__ MaxSum s_part[kCeThreads / 32];
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    MaxSum t = s_part[0];
#pragma unroll
    for (int w = 1; w < kCeThreads / 32; ++w) t = ms_merge(t, s_part[w]);
    // natural-log domain: logsumexp = m/log2e + ln(s)
    const float l = t.m * (1.0f / kLog2e) + logf(t.s);
    lse[row] = l;
    const int64_t tg = target[row];
    float rl = 0.f;
    if (tg != ignore_index && tg >= 0 && tg < vocab) rl = l - CeT<T>::ld(xr + tg);
    row_loss[row] = rl;
  }
}

// loss = sum(row_loss) / count(target != ignore_index)   (reduction 1 = mean, 2 = sum)
__global__ void __launch_bounds__(1024)
    k_ce_finish(float* __restrict__ loss, float* __restrict__ total_weight,
                const float* __restrict__ row_loss, const int64_t* __restrict__ target, int64_t rows,
                int64_t ignore_index, int reduction) {
  __shared__ float s_sum[1024];
  __shared__ float s_cnt[1024];
  float s = 0.f, c = 0.f;
  for (int64_t r = threadIdx.x; r < rows; r += 1024) {
    s += row_loss[r];
    c += (target[r] != ignore_index) ? 1.f : 0.f;
  }
  s_sum[threadIdx.x] = s;
  s_cnt[threadIdx.x] = c;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) {
      s_sum[threadIdx.x] += s_sum[threadIdx.x + o];
      s_cnt[threadIdx.x] += s_cnt[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    *total_weight = s_cnt[0];
    *loss = (reduction == 1) ? s_sum[0] / s_cnt[0] : s_sum[0];
  }
}

// dx[r, j] = c_r * (softmax(x_r)[j] - [j == target_r]),  c_r = grad_out / total_weight (mean) or
// grad_out (sum), 0 for ignored rows.  One CTA per row; padding columns [vocab, ld_out) are zeroed.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kCeThreads)
    k_ce_bwd(T* __restrict__ dx, int64_t ld_out, const T* __restrict__ x, int64_t ld,
             const int64_t* __restrict__ target, const float* __restrict__ lse,
             const float* __restrict__ grad_out, const float* __restrict__ total_weight,
             int64_t vocab, int64_t ignore_index, int reduction) {
  constexpr int EPV = CeT<T>::EPV;
  const int64_t row = blockIdx.x;
  const T* xr = x + row * ld;
  T* dr = dx + row * ld_out;
  const int64_t tg = target[row];
  float c = *grad_out;
  if (reduction == 1) c = c / *total_weight;
  if (tg == ignore_index) c = 0.f;
  const float nl = -lse[row] * kLog2e;
  if (VEC) {
    const int64_t nvec = vocab / EPV;
    const uint4* xv = reinterpret_cast<const uint4*>(xr);
    uint4* dv = reinterpret_cast<uint4*>(dr);
    const int64_t tvec = tg / EPV;
    const int te = (int)(tg - tvec * EPV);
    int64_t i = threadIdx.x;
    for (; i + 3 * kCeThreads < nvec; i += 4 * kCeThreads) {
      uint4 raw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) raw[u] = __ldg(xv + i + u * kCeThreads);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float f[8];
        CeT<T>::unpack(raw[u], f);
#pragma unroll
        for (int e = 0; e < EPV; ++e) {
          const float p = fast_exp2(fmaf(f[e], kLog2e, nl));
          f[e] = (i + u * kCeThreads == tvec && e == te) ? fmaf(p, c, -c) : p * c;
        }
        dv[i + u * kCeThreads] = CeT<T>::pack(f);
      }
    }
    for (; i < nvec; i += kCeThreads) {
      float f[8];
      CeT<T>::unpack(__ldg(xv + i), f);
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        const float p = fast_exp2(fmaf(f[e], kLog2e, nl));
        f[e] = (i == tvec && e == te) ? fmaf(p, c, -c) : p * c;
      }
      dv[i] = CeT<T>::pack(f);
    }
    for (int64_t j = nvec * EPV + threadIdx.x; j < ld_out; j += kCeThreads) {
      float v = 0.f;
      if (j < vocab) {
        const float p = fast_exp2(fmaf(CeT<T>::ld(xr + j), kLog2e, nl));
        v = (j == tg) ? fmaf(p, c, -c) : p * c;
      }
      CeT<T>::st(dr + j, v);
    }
  } else {
    for (int64_t j = threadIdx.x; j < ld_out; j += kCeThreads) {
      float v = 0.f;
      if (j < vocab) {
        const float p = fast_exp2(fmaf(CeT<T>::ld(xr + j), kLog2e, nl));
        v = (j == tg) ? fmaf(p, c, -c) : p * c;
      }
      CeT<T>::st(dr + j, v);
    }
  }
}

template <typename T>
static int ce_fwd_launch(float* lse, float* row_loss, const void* x, int64_t ld, const int64_t* target,
                         int64_t rows, int64_t vocab, int64_t ignore_index, cudaStream_t st) {
  const bool vec = (ld % CeT<T>::EPV == 0) && (((uintptr_t)x & 15) == 0);
  if (vec)
    k_ce_fwd<T, true><<<(unsigned)rows, kCeThreads, 0, st>>>(lse, row_loss, (const T*)x, ld, target, vocab,
                                                             ignore_index);
  else
    k_ce_fwd<T, false><<<(unsigned)rows, kCeThreads, 0, st>>>(lse, row_loss, (const T*)x, ld, target,
                                                              vocab, ignore_index);
  return EDB_OK;
}

template <typename T>
static int ce_bwd_launch(void* dx, int64_t ld_out, const void* x, int64_t ld, const int64_t* target,
                         const float* lse, const float* grad_out, const float* total_weight,
                         int64_t rows, int64_t vocab, int64_t ignore_index, int reduction,
                         cudaStream_t st) {
  const bool vec = (ld % CeT<T>::EPV == 0) && (ld_out % CeT<T>::EPV == 0) &&
                   ((((uintptr_t)x | (uintptr_t)dx) & 15) == 0);
  if (vec)
    k_ce_bwd<T, true><<<(unsigned)rows, kCeThreads, 0, st>>>((T*)dx, ld_out, (const T*)x, ld, target, lse,
                                                             grad_out, total_weight, vocab,
                                                             ignore_index, reduction);
  else
    k_ce_bwd<T, false><<<(unsigned)rows, kCeThreads, 0, st>>>((T*)dx, ld_out, (const T*)x, ld, target,
                                                              lse, grad_out, total_weight, vocab,
                                                              ignore_index, reduction);
  return EDB_OK;
}

}  // namespace edb

using namespace edb;

extern "C" {

int edb_cross_entropy_fwd(float* loss, float* total_weight, float* lse, float* row_loss,
                          const void* logits, int64_t ld, const int64_t* target, int64_t rows,
                          int64_t vocab, int64_t ignore_index, int reduction, int dtype, void* stream) {
  if (rows <= 0 || vocab <= 0 || rows > 0x7fffffffLL)
    return set_error(EDB_E_UNSUPPORTED, "edb_cross_entropy_fwd: rows=%lld vocab=%lld", (long long)rows,
                     (long long)vocab);
  if (reduction != 1 && reduction != 2)
    return set_error(EDB_E_UNSUPPORTED, "edb_cross_entropy_fwd: reduction %d (1 = mean, 2 = sum)", reduction);
  if (ld < vocab) return set_error(EDB_E_INVALID, "edb_cross_entropy_fwd: ld < vocab");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == EDB_BF16)
    ce_fwd_launch<__nv_bfloat16>(lse, row_loss, logits, ld, target, rows, vocab, ignore_index, st);
  else if (dtype == EDB_F32)
    ce_fwd_launch<float>(lse, row_loss, logits, ld, target, rows, vocab, ignore_index, st);
  else
    return set_error(EDB_E_UNSUPPORTED, "edb_cross_entropy_fwd: dtype %d", dtype);
  k_ce_finish<<<1, 1024, 0, st>>>(loss, total_weight, row_loss, target, rows, ignore_index, reduction);
  count_launch();
  count_launch();
  return cuda_check(cudaGetLastError(), "k_ce_fwd launch");
}

int edb_cross_entropy_bwd(void* dlogits, int64_t ld_out, const void* logits, int64_t ld,
                          const int64_t* target, const float* lse, const float* grad_out,
                          const float* total_weight, int64_t rows, int64_t vocab,
                          int64_t ignore_index, int reduction, int dtype, void* stream) {
  if (rows <= 0 || vocab <= 0 || rows > 0x7fffffffLL)
    return set_error(EDB_E_UNSUPPORTED, "edb_cross_entropy_bwd: rows=%lld vocab=%lld", (long long)rows,
                     (long long)vocab);
  if (reduction != 1 && reduction != 2)
    return set_error(EDB_E_UNSUPPORTED, "edb_cross_entropy_bwd: reduction %d (1 = mean, 2 = sum)", reduction);
  if (ld < vocab || ld_out < vocab) return set_error(EDB_E_INVALID, "edb_cross_entropy_bwd: ld < vocab");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == EDB_BF16)
    ce_bwd_launch<__nv_bfloat16>(dlogits, ld_out, logits, ld, target, lse, grad_out, total_weight, rows,
                                 vocab, ignore_index, reduction, st);
  else if (dtype == EDB_F32)
    ce_bwd_launch<float>(dlogits, ld_out, logits, ld, target, lse, grad_out, total_weight, rows, vocab,
                         ignore_index, reduction, st);
  else
    return set_error(EDB_E_UNSUPPORTED, "edb_cross_entropy_bwd: dtype %d", dtype);
  count_launch();
  return cuda_check(cudaGetLastError(), "k_ce_bwd launch");
}

}  // extern "C"
