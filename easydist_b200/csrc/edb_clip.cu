// Multi-tensor kernels of gradient-norm clipping, `torch.nn.utils.clip_grad_norm_(params, max_norm)`
// with norm_type 2.  Traced, the clip is one linalg_vector_norm per gradient, a stack, the total norm
// and a coefficient, then one in-place mul_ per gradient: three passes over every gradient and about
// 2T + 6 launches for T parameters.
//
//   edb_grad_sumsq   sum of squares (or the norm) of every tensor of a list in one read: each CTA
//                    reduces one chunk of one tensor (chunks never straddle tensors) into one fp32
//                    partial; a finish kernel adds each tensor's partials in index order.  No atomics,
//                    so the result is deterministic and the pair can be captured in a CUDA graph.
//   edb_multi_scale_ g = T(g*c) in place over a list, the rounding of ATen's mul_ (for optimizers that
//                    are not fused here; the fused SGD takes the coefficient itself, edb_optim.cu).
#include <cuda_bf16.h>

#include "edb_internal.cuh"
#include "edb_vec.cuh"

namespace edb {

constexpr int kClipMaxTensors = 320;  // per launch; descriptors travel as kernel parameters
constexpr int kClipThreads = 256;
constexpr int kClipUnroll = 4;        // 16-byte vectors per thread and chunk
constexpr int kClipWarps = kClipThreads / 32;

struct ClipTensor {
  void* p;
  int64_t numel;
};
struct ClipDesc {
  ClipTensor t[kClipMaxTensors];
  int first_chunk[kClipMaxTensors + 1];  // prefix sum of chunks per tensor
  int n;
};
static_assert(sizeof(ClipDesc) <= 16 * 1024, "descriptor must fit the kernel parameter space");

template <typename T> __host__ __device__ constexpr int64_t chunk_elems() {
  return (int64_t)kClipThreads * kClipUnroll * VecT<T>::EPV;
}

// tensor of chunk c: the last index whose first chunk is <= c (empty tensors own no chunk)
__device__ __forceinline__ int chunk_owner(const ClipDesc& d, int c) {
  int lo = 0, hi = d.n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (d.first_chunk[mid] <= c) lo = mid;
    else hi = mid;
  }
  return lo;
}

// fixed-order CTA sum: a 5-level shuffle tree per warp, then warp 0..7 added in sequence by thread 0
__device__ __forceinline__ float block_sum(float v) {
  __shared__ float warp_sum[kClipWarps];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0) {
    s = warp_sum[0];
#pragma unroll
    for (int w = 1; w < kClipWarps; ++w) s += warp_sum[w];
  }
  return s;  // valid in thread 0
}

// One chunk of one tensor -> partial[c].  A thread adds its squares in sequence: the 16-byte vectors
// u = 0..3 element by element, then (last chunk of an aligned tensor) one tail element.  Tensors whose
// address is not 16-byte aligned are read element by element over the same chunk.
template <typename T>
__global__ void __launch_bounds__(kClipThreads)
    k_grad_sumsq_partial(const __grid_constant__ ClipDesc d, float* __restrict__ partial) {
  constexpr int EPV = VecT<T>::EPV;
  constexpr int64_t CE = chunk_elems<T>();
  const int c = (int)blockIdx.x;
  const int ti = chunk_owner(d, c);
  const ClipTensor& t = d.t[ti];
  const int64_t e0 = (int64_t)(c - d.first_chunk[ti]) * CE;
  const int64_t e1 = min(e0 + CE, t.numel);
  float acc = 0.f;
  if (((uintptr_t)t.p & 15) == 0) {
    const uint4* v = reinterpret_cast<const uint4*>(t.p);
    const int64_t nvec = t.numel / EPV;
    const int64_t v0 = e0 / EPV;
    uint4 r[kClipUnroll];
#pragma unroll
    for (int u = 0; u < kClipUnroll; ++u) {
      const int64_t i = v0 + u * kClipThreads + threadIdx.x;
      if (i < nvec) r[u] = __ldg(v + i);
    }
#pragma unroll
    for (int u = 0; u < kClipUnroll; ++u) {
      const int64_t i = v0 + u * kClipThreads + threadIdx.x;
      if (i < nvec) {
        float f[EPV];
        VecT<T>::unpack(r[u], f);
#pragma unroll
        for (int e = 0; e < EPV; ++e) acc = fmaf(f[e], f[e], acc);
      }
    }
    const int64_t tail = nvec * EPV + threadIdx.x;  // numel % EPV < EPV <= threads
    if (tail >= e0 && tail < e1) {
      const float x = VecT<T>::ld(reinterpret_cast<const T*>(t.p) + tail);
      acc = fmaf(x, x, acc);
    }
  } else {
    const T* p = reinterpret_cast<const T*>(t.p);
    for (int64_t i = e0 + threadIdx.x; i < e1; i += kClipThreads) {
      const float x = VecT<T>::ld(p + i);
      acc = fmaf(x, x, acc);
    }
  }
  const float s = block_sum(acc);
  if (threadIdx.x == 0) partial[c] = s;
}

// One CTA per tensor: thread k adds partials k, k+256, ... in sequence, then block_sum.
// raw: out[i] = sum (fp32); else out[i] = T(sqrtf(sum)), what linalg_vector_norm(g, 2) returns.
template <typename T>
__global__ void __launch_bounds__(kClipThreads)
    k_grad_sumsq_finish(const __grid_constant__ ClipDesc d, const float* __restrict__ partial,
                        void* __restrict__ out, int raw) {
  const int i = (int)blockIdx.x;
  float acc = 0.f;
  for (int k = d.first_chunk[i] + (int)threadIdx.x; k < d.first_chunk[i + 1]; k += kClipThreads)
    acc += partial[k];
  const float s = block_sum(acc);
  if (threadIdx.x == 0) {
    if (raw) reinterpret_cast<float*>(out)[i] = s;
    else VecT<T>::st(reinterpret_cast<T*>(out) + i, sqrtf(s));
  }
}

// g = T(g*c) in place, one chunk per CTA (same geometry as k_grad_sumsq_partial)
template <typename T>
__global__ void __launch_bounds__(kClipThreads)
    k_multi_scale(const __grid_constant__ ClipDesc d, const T* __restrict__ coef) {
  constexpr int EPV = VecT<T>::EPV;
  constexpr int64_t CE = chunk_elems<T>();
  const int c = (int)blockIdx.x;
  const int ti = chunk_owner(d, c);
  const ClipTensor& t = d.t[ti];
  const int64_t e0 = (int64_t)(c - d.first_chunk[ti]) * CE;
  const int64_t e1 = min(e0 + CE, t.numel);
  const float cf = VecT<T>::ld(coef);
  T* p = reinterpret_cast<T*>(t.p);
  if (((uintptr_t)t.p & 15) == 0) {
    uint4* v = reinterpret_cast<uint4*>(t.p);
    const int64_t nvec = t.numel / EPV;
    const int64_t v0 = e0 / EPV;
    uint4 r[kClipUnroll];
#pragma unroll
    for (int u = 0; u < kClipUnroll; ++u) {
      const int64_t i = v0 + u * kClipThreads + threadIdx.x;
      if (i < nvec) r[u] = v[i];
    }
#pragma unroll
    for (int u = 0; u < kClipUnroll; ++u) {
      const int64_t i = v0 + u * kClipThreads + threadIdx.x;
      if (i < nvec) {
        float f[EPV];
        VecT<T>::unpack(r[u], f);
#pragma unroll
        for (int e = 0; e < EPV; ++e) f[e] = __fmul_rn(f[e], cf);
        v[i] = VecT<T>::pack(f);
      }
    }
    const int64_t tail = nvec * EPV + threadIdx.x;
    if (tail >= e0 && tail < e1) VecT<T>::st(p + tail, __fmul_rn(VecT<T>::ld(p + tail), cf));
  } else {
    for (int64_t i = e0 + threadIdx.x; i < e1; i += kClipThreads)
      VecT<T>::st(p + i, __fmul_rn(VecT<T>::ld(p + i), cf));
  }
}

// Split the list into launches of at most kClipMaxTensors tensors (and 2^31-1 chunks) and call
// launch(desc, chunks, first tensor, first chunk overall) for each.  Arguments are checked first.
template <typename F>
int for_each_launch(const char* who, int n, void* const* ptrs, const int64_t* numels, int dtype,
                    F launch) {
  if (n < 0 || (n > 0 && (ptrs == nullptr || numels == nullptr)))
    return set_error(EDB_E_INVALID, "%s: bad tensor list", who);
  if (dtype != EDB_BF16 && dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "%s: dtype %d", who, dtype);
  const int64_t ce = dtype == EDB_BF16 ? chunk_elems<__nv_bfloat16>() : chunk_elems<float>();
  for (int i = 0; i < n; ++i) {
    if (numels[i] < 0) return set_error(EDB_E_INVALID, "%s: negative numel (tensor %d)", who, i);
    if (numels[i] > 0 && ptrs[i] == nullptr)
      return set_error(EDB_E_INVALID, "%s: null pointer (tensor %d)", who, i);
    if ((numels[i] + ce - 1) / ce > 0x7fffffffLL)
      return set_error(EDB_E_UNSUPPORTED, "%s: tensor %d too large", who, i);
  }
  int done = 0;
  int64_t chunk_base = 0;
  while (done < n) {
    ClipDesc d;
    int k = 0;
    int64_t chunks = 0;
    d.first_chunk[0] = 0;
    const int first = done;
    while (done < n && k < kClipMaxTensors) {
      const int64_t c = (numels[done] + ce - 1) / ce;
      if (chunks + c > 0x7fffffffLL) break;
      d.t[k].p = ptrs[done];
      d.t[k].numel = numels[done];
      chunks += c;
      d.first_chunk[++k] = (int)chunks;
      ++done;
    }
    d.n = k;
    const int rc = launch(d, chunks, first, chunk_base);
    if (rc != EDB_OK) return rc;
    chunk_base += chunks;
  }
  return EDB_OK;
}

}  // namespace edb

using namespace edb;

extern "C" {

int edb_grad_sumsq_workspace(int n, const int64_t* numels, int dtype, size_t* bytes_out) {
  if (bytes_out == nullptr || n < 0 || (n > 0 && numels == nullptr))
    return set_error(EDB_E_INVALID, "edb_grad_sumsq_workspace: bad arguments");
  if (dtype != EDB_BF16 && dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "edb_grad_sumsq_workspace: dtype %d", dtype);
  const int64_t ce = dtype == EDB_BF16 ? chunk_elems<__nv_bfloat16>() : chunk_elems<float>();
  int64_t chunks = 0;
  for (int i = 0; i < n; ++i) {
    if (numels[i] < 0) return set_error(EDB_E_INVALID, "edb_grad_sumsq_workspace: negative numel");
    chunks += (numels[i] + ce - 1) / ce;
  }
  *bytes_out = (size_t)chunks * sizeof(float);
  return EDB_OK;
}

int edb_grad_sumsq(int n, const void* const* grads, const int64_t* numels, void* out,
                   void* workspace, int mode, int dtype, void* stream) {
  if (mode != EDB_SUMSQ_RAW && mode != EDB_SUMSQ_NORM)
    return set_error(EDB_E_INVALID, "edb_grad_sumsq: mode %d", mode);
  if (n > 0 && out == nullptr) return set_error(EDB_E_INVALID, "edb_grad_sumsq: out is NULL");
  size_t need = 0;
  if (n > 0) {
    const int rc = edb_grad_sumsq_workspace(n, numels, dtype, &need);
    if (rc != EDB_OK) return rc;
  }
  if (need > 0 && workspace == nullptr)
    return set_error(EDB_E_INVALID, "edb_grad_sumsq: workspace is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  const int raw = mode == EDB_SUMSQ_RAW;
  const size_t out_elem = raw ? sizeof(float) : (dtype == EDB_BF16 ? 2 : 4);
  float* partial = reinterpret_cast<float*>(workspace);
  const int rc = for_each_launch(
      "edb_grad_sumsq", n, const_cast<void* const*>(grads), numels, dtype,
      [&](const ClipDesc& d, int64_t chunks, int first, int64_t chunk_base) {
        void* o = reinterpret_cast<char*>(out) + (size_t)first * out_elem;
        float* part = partial + chunk_base;
        if (dtype == EDB_BF16) {
          if (chunks > 0) k_grad_sumsq_partial<__nv_bfloat16><<<(unsigned)chunks, kClipThreads, 0, st>>>(d, part);
          k_grad_sumsq_finish<__nv_bfloat16><<<d.n, kClipThreads, 0, st>>>(d, part, o, raw);
        } else {
          if (chunks > 0) k_grad_sumsq_partial<float><<<(unsigned)chunks, kClipThreads, 0, st>>>(d, part);
          k_grad_sumsq_finish<float><<<d.n, kClipThreads, 0, st>>>(d, part, o, raw);
        }
        count_launch();
        if (chunks > 0) count_launch();
        return EDB_OK;
      });
  if (rc != EDB_OK) return rc;
  return cuda_check(cudaGetLastError(), "k_grad_sumsq launch");
}

int edb_multi_scale_(int n, void* const* grads, const int64_t* numels, const void* coef, int dtype,
                     void* stream) {
  if (n > 0 && coef == nullptr) return set_error(EDB_E_INVALID, "edb_multi_scale_: coef is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = for_each_launch(
      "edb_multi_scale_", n, grads, numels, dtype,
      [&](const ClipDesc& d, int64_t chunks, int, int64_t) {
        if (chunks == 0) return EDB_OK;
        if (dtype == EDB_BF16)
          k_multi_scale<__nv_bfloat16><<<(unsigned)chunks, kClipThreads, 0, st>>>(
              d, reinterpret_cast<const __nv_bfloat16*>(coef));
        else
          k_multi_scale<float><<<(unsigned)chunks, kClipThreads, 0, st>>>(
              d, reinterpret_cast<const float*>(coef));
        count_launch();
        return EDB_OK;
      });
  if (rc != EDB_OK) return rc;
  return cuda_check(cudaGetLastError(), "k_multi_scale launch");
}

}  // extern "C"
