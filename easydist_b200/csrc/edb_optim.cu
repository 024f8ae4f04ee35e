// Fused multi-tensor SGD-momentum update for the optimizer region of the compiled train step.
//
// The reference traces the optimizer into the same graph as forward and backward
// (easydist/torch/compile_auto.py:262-318 / compile_dp.py:201-260: params, grads and optimizer states
// are graph values), so its update shows up as foreach nodes.  After re-inplacing, torch.optim.SGD
// (momentum, foreach=True) is three of them:
//     _foreach_mul_(bufs, mu); _foreach_add_(bufs, grads, alpha=1-dampening);
//     _foreach_add_(params, bufs, alpha=-lr)
// = 36 + 18 multi_tensor_apply launches moving 7 x sizeof(model) bytes (bufs twice read + twice
// written, params and grads once each...).  One pass needs 5 x sizeof(model): read p, g, m; write
// p, m.  This kernel does that pass for every tensor of the lists in one launch (up to
// kOptMaxTensors per launch), 16-byte vector accesses, and reproduces the rounding of the three
// ATen ops exactly (each op computes in fp32 and rounds to the storage dtype), so the result is
// bit-identical to the unfused graph.
#include <cuda_bf16.h>

#include "edb_internal.cuh"
#include "edb_vec.cuh"

namespace edb {

constexpr int kOptMaxTensors = 320;     // per launch; descriptors travel as kernel parameters
constexpr int kOptThreads = 256;
constexpr int kOptChunkVecs = 4 * kOptThreads;  // 16-byte vectors per CTA

struct OptTensor {
  void* p;
  const void* g;
  void* m;
  int64_t numel;
};
struct OptDesc {
  OptTensor t[kOptMaxTensors];
  int first_chunk[kOptMaxTensors + 1];  // prefix sum of chunks per tensor
  int n;
  float mu, grad_alpha, neg_lr;
  const void* grad_scale;  // kScaled: device scalar c of the storage dtype
};
static_assert(sizeof(OptDesc) <= 16 * 1024, "descriptor must fit the kernel parameter space");

template <typename T> using OptT = VecT<T>;

// the three ATen ops, one element: every op rounds to the storage dtype
template <typename T>
__device__ __forceinline__ void sgd_elem(float& p, float g, float& m, float mu, float ga, float nlr) {
  const float t = OptT<T>::rnd(m * mu);            // _foreach_mul_(bufs, mu)
  m = OptT<T>::rnd(fmaf(ga, g, t));                // _foreach_add_(bufs, grads, alpha=ga)
  p = OptT<T>::rnd(fmaf(nlr, m, p));               // _foreach_add_(params, bufs, alpha=-lr)
}

// kScaled: g' = T(g*c) first, the rounding of the in-place `mul_(g, c)` of gradient clipping
template <typename T, bool kScaled>
__global__ void __launch_bounds__(kOptThreads)
    k_sgd_momentum(const __grid_constant__ OptDesc d) {
  constexpr int EPV = OptT<T>::EPV;
  // which tensor does this chunk belong to (binary search over the prefix sums)
  int lo = 0, hi = d.n;
  const int c = (int)blockIdx.x;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (d.first_chunk[mid] <= c) lo = mid;
    else hi = mid;
  }
  const OptTensor& t = d.t[lo];
  const int64_t v0 = (int64_t)(c - d.first_chunk[lo]) * kOptChunkVecs;
  const int64_t nvec = t.numel / EPV;
  uint4* pv = reinterpret_cast<uint4*>(t.p);
  const uint4* gv = reinterpret_cast<const uint4*>(t.g);
  uint4* mv = reinterpret_cast<uint4*>(t.m);
  const float mu = d.mu, ga = d.grad_alpha, nlr = d.neg_lr;
  const float gc = kScaled ? OptT<T>::ld(reinterpret_cast<const T*>(d.grad_scale)) : 1.f;
  uint4 rp[4], rg[4], rm[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int64_t i = v0 + u * kOptThreads + threadIdx.x;
    if (i < nvec) {
      rp[u] = pv[i];
      rg[u] = __ldg(gv + i);
      rm[u] = mv[i];
    }
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int64_t i = v0 + u * kOptThreads + threadIdx.x;
    if (i < nvec) {
      float fp[EPV], fg[EPV], fm[EPV];
      OptT<T>::unpack(rp[u], fp);
      OptT<T>::unpack(rg[u], fg);
      OptT<T>::unpack(rm[u], fm);
      if (kScaled) {
#pragma unroll
        for (int e = 0; e < EPV; ++e) fg[e] = OptT<T>::rnd(__fmul_rn(fg[e], gc));
      }
#pragma unroll
      for (int e = 0; e < EPV; ++e) sgd_elem<T>(fp[e], fg[e], fm[e], mu, ga, nlr);
      mv[i] = OptT<T>::pack(fm);
      pv[i] = OptT<T>::pack(fp);
    }
  }
  // scalar tail (numel % EPV elements), done by the tensor's last chunk
  const int64_t tail0 = nvec * EPV;
  if (v0 + kOptChunkVecs >= nvec && tail0 + threadIdx.x < t.numel) {
    const int64_t i = tail0 + threadIdx.x;
    T* p = reinterpret_cast<T*>(t.p) + i;
    T* m = reinterpret_cast<T*>(t.m) + i;
    float fp = OptT<T>::ld(p), fm = OptT<T>::ld(m);
    float fg = OptT<T>::ld(reinterpret_cast<const T*>(t.g) + i);
    if (kScaled) fg = OptT<T>::rnd(__fmul_rn(fg, gc));
    sgd_elem<T>(fp, fg, fm, mu, ga, nlr);
    OptT<T>::st(m, fm);
    OptT<T>::st(p, fp);
  }
}

}  // namespace edb

using namespace edb;

extern "C" {

static int sgd_momentum(int n, void* const* params, const void* const* grads, void* const* bufs,
                        const int64_t* numels, float mu, float grad_alpha, float neg_lr,
                        const void* grad_scale, int dtype, void* stream) {
  if (n <= 0) return EDB_OK;
  if (dtype != EDB_BF16 && dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "edb_sgd_momentum: dtype %d", dtype);
  const int epv = dtype == EDB_BF16 ? 8 : 4;
  for (int i = 0; i < n; ++i) {
    if (numels[i] < 0) return set_error(EDB_E_INVALID, "edb_sgd_momentum: negative numel");
    if (((uintptr_t)params[i] | (uintptr_t)grads[i] | (uintptr_t)bufs[i]) & 15)
      return set_error(EDB_E_UNSUPPORTED, "edb_sgd_momentum: tensor %d is not 16-byte aligned", i);
  }
  cudaStream_t st = (cudaStream_t)stream;
  int done = 0;
  while (done < n) {
    OptDesc d;
    d.mu = mu;
    d.grad_alpha = grad_alpha;
    d.neg_lr = neg_lr;
    d.grad_scale = grad_scale;
    int k = 0;
    int64_t chunks = 0;
    d.first_chunk[0] = 0;
    while (done < n && k < kOptMaxTensors) {
      const int64_t numel = numels[done];
      if (numel > 0) {
        const int64_t nvec = numel / epv;
        int64_t c = (nvec + kOptChunkVecs - 1) / kOptChunkVecs;
        if (c == 0) c = 1;  // tail-only tensor
        if (chunks + c > 0x7fffffffLL) break;
        d.t[k].p = params[done];
        d.t[k].g = grads[done];
        d.t[k].m = bufs[done];
        d.t[k].numel = numel;
        chunks += c;
        d.first_chunk[++k] = (int)chunks;
      }
      ++done;
    }
    d.n = k;
    if (k == 0) {
      if (done < n) return set_error(EDB_E_UNSUPPORTED, "edb_sgd_momentum: tensor %d too large", done);
      continue;
    }
    const unsigned grid = (unsigned)chunks;
    if (dtype == EDB_BF16) {
      if (grad_scale) k_sgd_momentum<__nv_bfloat16, true><<<grid, kOptThreads, 0, st>>>(d);
      else k_sgd_momentum<__nv_bfloat16, false><<<grid, kOptThreads, 0, st>>>(d);
    } else {
      if (grad_scale) k_sgd_momentum<float, true><<<grid, kOptThreads, 0, st>>>(d);
      else k_sgd_momentum<float, false><<<grid, kOptThreads, 0, st>>>(d);
    }
    count_launch();
  }
  return cuda_check(cudaGetLastError(), "k_sgd_momentum launch");
}

int edb_sgd_momentum(int n, void* const* params, const void* const* grads, void* const* bufs,
                     const int64_t* numels, float mu, float grad_alpha, float neg_lr, int dtype,
                     void* stream) {
  return sgd_momentum(n, params, grads, bufs, numels, mu, grad_alpha, neg_lr, nullptr, dtype, stream);
}

int edb_sgd_momentum_scaled(int n, void* const* params, const void* const* grads, void* const* bufs,
                            const int64_t* numels, float mu, float grad_alpha, float neg_lr,
                            const void* grad_scale, int dtype, void* stream) {
  if (n > 0 && grad_scale == nullptr)
    return set_error(EDB_E_INVALID, "edb_sgd_momentum_scaled: grad_scale is NULL");
  return sgd_momentum(n, params, grads, bufs, numels, mu, grad_alpha, neg_lr, grad_scale, dtype,
                      stream);
}

}  // extern "C"
