// Scaled-dot-product attention on Hopper tensor cores (wgmma + TMA + mbarrier): bf16 q, k, v of one
// shape [B, H, T, hd], hd 64 or 128, causal or not, fp32 accumulation and softmax statistics.
//
// Every kernel is one CTA of 384 threads: two consumer warpgroups that each own 64 rows of the
// CTA's 128-row block, and a producer warpgroup whose first thread TMA-loads the tiles the consumers stream
// through a two-stage shared-memory ring (full / empty mbarriers, one empty arrive per warpgroup).
// Tiles are read where they lie through 4-D tensor maps over (hd, T, H, B): a strided view (the
// c_attn split, a transposed projection) costs no copy, and rows past T arrive as zeros.  A tile of
// R rows is hd / 64 boxes of R x 64 elements in the 128-byte-swizzle layout, so one tile serves as a
// K-major operand (contracting over hd) and as an MN-major B operand (contracting over its rows).
//
// Forward (flash attention): S = Q·Kᵀ (both operands in shared memory), online softmax in registers
// in the log2 domain (scale·log2e folded into one FMA, exp2), P rounded to bf16 and fed from
// registers to O += P·V.  Only tiles that cross the diagonal or T are masked.  Writes O (bf16) and
// the natural-log logsumexp (fp32).
//
// Backward, deterministic (no float atomics): every output element is summed by one thread in a
// fixed order.
//   prep : D = rowsum(dO∘O) and lse·log2e into a workspace padded to 128 rows (pad: D = 0,
//          lse = +inf, so padded query rows carry P = 0)
//   dK/dV: one CTA per 128 key rows; per 64 query rows Sᵀ = K·Qᵀ, Pᵀ = exp2(Sᵀ·c - lse),
//          dV += Pᵀ·dO, dPᵀ = V·dOᵀ, dSᵀ = Pᵀ∘(dPᵀ - D), dK += dSᵀ·Q
//   dQ   : one CTA per 128 query rows; per 64 key rows S, P, dP = dO·Vᵀ, dS, dQ += dS·K
// P is rounded to bf16 before it multiplies dO and before dS; dS is rounded to bf16.  Seven
// matmuls per tile pair instead of the five of an atomic dQ.
#include <cuda.h>
#include <cuda_bf16.h>
#include <math.h>

#include "edb_internal.cuh"
#include "edb_sm90.cuh"

namespace edb {
namespace {

// two consumer warpgroups + a producer warpgroup that hands its registers to them: a 384-thread
// CTA starts at 168 registers a thread, the consumers grow to 232 (dK and dV of hd 128 are 128 fp32
// accumulators a thread) and the producer shrinks to 40.
constexpr int kAttnThreads = 384;
constexpr int kStages = 2;
constexpr int kPad = 128;          // workspace rows per (b, h) are padded to a multiple of this
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

struct Rows {            // element strides of a [B, H, T, hd] operand (hd stride 1)
  int64_t b, h, t;
};

__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~static_cast<uintptr_t>(1023));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t u) {
  return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
}
__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// The 64 rows from row0 of an R-row tile as a K-major operand, k step kk (16 of the hd columns).
template <int R>
__device__ __forceinline__ uint64_t desc_k(uint32_t tile, int row0, int kk) {
  return make_smem_desc(tile + (kk >> 2) * R * 128 + row0 * 128 + (kk & 3) * 32, 16, 1024);
}
// An R-row tile as an MN-major B operand (N = hd): k step kk = its rows [16 kk, 16 kk + 16).
template <int R>
__device__ __forceinline__ uint64_t desc_mn(uint32_t tile, int kk) {
  return make_smem_desc(tile + kk * 16 * 128, R * 128, 1024);
}

// acc[64 x HD] += A[64 x 16 kk_count] (registers, 4 per k step) · tile (MN-major), R-row tile.
template <int HD, int R>
__device__ __forceinline__ void mma_rs(float* acc, const uint32_t* a, uint32_t tile) {
#pragma unroll
  for (int kk = 0; kk < R / 16; ++kk) {
    if constexpr (HD == 128) wgmma_m64n128k16_rs<1>(acc, a + 4 * kk, desc_mn<R>(tile, kk), 1u);
    else wgmma_m64n64k16_rs<1>(acc, a + 4 * kk, desc_mn<R>(tile, kk), 1u);
  }
}

// acc[64 x N] = rows [row0, row0 + 64) of an RA-row tile · (an N-row tile)ᵀ, both K-major over hd.
template <int HD, int N, int RA>
__device__ __forceinline__ void mma_ss(float* acc, uint32_t a, int row0, uint32_t b) {
#pragma unroll
  for (int kk = 0; kk < HD / 16; ++kk) {
    if constexpr (N == 128) wgmma_m64n128k16<0, 0>(acc, desc_k<RA>(a, row0, kk), desc_k<N>(b, 0, kk), kk > 0);
    else wgmma_m64n64k16<0, 0>(acc, desc_k<RA>(a, row0, kk), desc_k<N>(b, 0, kk), kk > 0);
  }
}

template <int HD, int R>
__device__ __forceinline__ void load_tile(const CUtensorMap* map, uint64_t* bar, uint8_t* dst, int row,
                                          int h, int b) {
#pragma unroll
  for (int c = 0; c < HD / 64; ++c) tma_load_4d(map, bar, dst + c * R * 128, c * 64, row, h, b);
}

// Store this thread's rows of a 64 x HD fp32 fragment, times `mul`, as bf16 (rows < T only).
template <int HD>
__device__ __forceinline__ void store_rows(__nv_bfloat16* base, const Rows& st, int b, int h, int r0,
                                           int T, int c0, const float* acc, const float* mul) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = r0 + 8 * hh;
    if (row >= T) continue;
    __nv_bfloat16* p = base + b * st.b + h * st.h + row * st.t + c0;
#pragma unroll
    for (int j = 0; j < HD / 8; ++j) {
      const int i = 4 * j + 2 * hh;
      *reinterpret_cast<uint32_t*>(p + 8 * j) = pack_bf16(acc[i] * mul[hh], acc[i + 1] * mul[hh]);
    }
  }
}

// ---- forward -----------------------------------------------------------------------------------------

struct FwdArgs {
  __nv_bfloat16* o;
  float* lse;
  Rows os, ls;
  int T, causal;
  float scale_log2;
};

template <int HD> struct FwdCfg {
  static constexpr int BM = 128, BN = 128;
  static constexpr int kQBytes = BM * HD * 2;
  static constexpr int kKVBytes = BN * HD * 2;  // K or V of one stage
  static constexpr int kSmemBytes = kQBytes + kStages * 2 * kKVBytes + 1024 + 256;
};

template <int HD>
__global__ void __launch_bounds__(kAttnThreads, 1)
    k_attn_fwd(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
               const __grid_constant__ CUtensorMap tv, const FwdArgs a) {
  using C = FwdCfg<HD>;
  constexpr int BM = C::BM, BN = C::BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sq = align1024(smem_raw);
  uint8_t* skv = sq + C::kQBytes;  // stage s: K at skv + 2 s kKVBytes, V behind it
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(skv + kStages * 2 * C::kKVBytes);
  uint64_t* full = q_bar + 1;
  uint64_t* empty = full + kStages;

  const int m_blocks = (a.T + BM - 1) / BM;
  const int mb = a.causal ? m_blocks - 1 - (int)blockIdx.x : (int)blockIdx.x;  // longest rows first
  const int h = blockIdx.y, b = blockIdx.z, m0 = mb * BM;
  const int n_all = (a.T + BN - 1) / BN;
  const int n_blocks = a.causal ? min(n_all, (m0 + BM + BN - 1) / BN) : n_all;

  if (threadIdx.x == 0) {
    mbar_init(q_bar, 1);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  bool ok = true;  // false: a barrier wait ran into the watchdog
  const int warp = threadIdx.x >> 5;
  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 256) {
      prefetch_tmap(&tq);
      prefetch_tmap(&tk);
      prefetch_tmap(&tv);
      mbar_expect_tx(q_bar, C::kQBytes);
      load_tile<HD, BM>(&tq, q_bar, sq, m0, h, b);
      for (int n = 0; n < n_blocks; ++n) {
        const int s = n % kStages;
        if (!(ok = mbar_wait_ok(&empty[s], ((n / kStages) & 1) ^ 1))) break;
        mbar_expect_tx(&full[s], 2 * C::kKVBytes);
        uint8_t* sk = skv + s * 2 * C::kKVBytes;
        load_tile<HD, BN>(&tk, &full[s], sk, n * BN, h, b);
        load_tile<HD, BN>(&tv, &full[s], sk + C::kKVBytes, n * BN, h, b);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const int r0 = m0 + wg * 64 + 16 * (t >> 5) + ((t & 31) >> 2);  // this thread's rows: r0, r0 + 8
    const int c0 = 2 * (t & 3);
    const float sl2 = a.scale_log2;
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const uint32_t q_addr = smem_u32(sq);
    ok = mbar_wait_ok(q_bar, 0);

    for (int n = 0; ok && n < n_blocks; ++n) {
      const int s = n % kStages;
      const uint32_t k_addr = smem_u32(skv + s * 2 * C::kKVBytes), v_addr = k_addr + C::kKVBytes;
      if (!(ok = mbar_wait_ok(&full[s], (n / kStages) & 1))) break;
      float sc[BN / 2];
      wgmma_fence();
      mma_ss<HD, BN, BM>(sc, q_addr, wg * 64, k_addr);
      wgmma_commit();
      wgmma_wait<0>();

      const int n0 = n * BN;
      if ((a.causal && n0 + BN - 1 > m0 + wg * 64) || n0 + BN > a.T) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) {
          const int col = n0 + 8 * (i >> 2) + c0 + (i & 1), row = r0 + 8 * ((i >> 1) & 1);
          if (col >= a.T || (a.causal && col > row)) sc[i] = -INFINITY;
        }
      }
      float base[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = m_run[hh];
#pragma unroll
        for (int i = 2 * hh; i < BN / 2; i += 4) mx = fmaxf(mx, fmaxf(sc[i], sc[i + 1]));
        mx = quad_max(mx);
        base[hh] = mx == -INFINITY ? 0.f : mx * sl2;  // a row with nothing visible yet keeps P = 0
        const float alpha = exp2f(m_run[hh] * sl2 - base[hh]);
        m_run[hh] = mx;
        l_run[hh] *= alpha;
#pragma unroll
        for (int i = 2 * hh; i < HD / 2; i += 4) {
          o[i] *= alpha;
          o[i + 1] *= alpha;
        }
      }
      uint32_t p[BN / 4];
#pragma unroll
      for (int i = 0; i < BN / 2; i += 2) {
        const int hh = (i >> 1) & 1;
        const float p0 = exp2f(fmaf(sc[i], sl2, -base[hh])), p1 = exp2f(fmaf(sc[i + 1], sl2, -base[hh]));
        l_run[hh] += p0 + p1;
        p[i >> 1] = pack_bf16(p0, p1);
      }
      wgmma_fence();
      mma_rs<HD, BN>(o, p, v_addr);
      wgmma_commit();
      wgmma_wait<0>();
      if (t == 0) mbar_arrive(&empty[s]);
    }

    float inv[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      l_run[hh] = quad_sum(l_run[hh]);
      inv[hh] = l_run[hh] > 0.f ? 1.f / l_run[hh] : 0.f;
    }
    store_rows<HD>(a.o, a.os, b, h, r0, a.T, c0, o, inv);
    if ((t & 3) == 0) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = r0 + 8 * hh;
        if (row < a.T)
          a.lse[b * a.ls.b + h * a.ls.h + row * a.ls.t] =
              l_run[hh] > 0.f ? (m_run[hh] * sl2 + log2f(l_run[hh])) * kLn2 : -INFINITY;
      }
    }
  }
  if (!ok) asm volatile("trap;");  // a protocol bug becomes a launch error, not a hung GPU
}

// ---- backward ----------------------------------------------------------------------------------------

struct BwdArgs {
  __nv_bfloat16 *dq, *dk, *dv;
  const __nv_bfloat16 *dout, *out;
  const float* lse;
  float* ws;  // [2][B H][Tp]: lse·log2e, then D
  Rows dos, outs, ls, dqs, dks, dvs;
  int T, Tp, H, causal;
  float scale, scale_log2;
};

// One warp per (b, h, row) of the padded workspace.
template <int HD>
__global__ void __launch_bounds__(256) k_attn_bwd_prep(const BwdArgs a, int64_t rows) {
  const int64_t idx = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (idx >= rows) return;
  const int64_t bh = idx / a.Tp;
  const int r = (int)(idx % a.Tp), b = (int)(bh / a.H), h = (int)(bh % a.H);
  float d = 0.f, l2 = INFINITY;
  if (r < a.T) {
    constexpr int V = HD / 32;
    const __nv_bfloat16* po = a.out + b * a.outs.b + h * a.outs.h + r * a.outs.t + lane * V;
    const __nv_bfloat16* pd = a.dout + b * a.dos.b + h * a.dos.h + r * a.dos.t + lane * V;
#pragma unroll
    for (int j = 0; j < V; ++j) d = fmaf(__bfloat162float(po[j]), __bfloat162float(pd[j]), d);
#pragma unroll
    for (int w = 16; w > 0; w >>= 1) d += __shfl_xor_sync(0xffffffffu, d, w);
    l2 = a.lse[b * a.ls.b + h * a.ls.h + r * a.ls.t] * kLog2e;
  }
  if (lane == 0) {
    a.ws[idx] = l2;
    a.ws[rows + idx] = d;
  }
}

template <int HD> struct DkdvCfg {
  static constexpr int BN = 128, BM = 64;       // key rows per CTA, query rows per step
  static constexpr int kKVBytes = BN * HD * 2;  // K or V
  static constexpr int kQBytes = BM * HD * 2;   // Q or dO of one stage
  static constexpr int kVecBytes = BM * 4;      // lse·log2e or D of one stage
  static constexpr int kSmemBytes = 2 * kKVBytes + kStages * (2 * kQBytes + 2 * kVecBytes) + 1024 + 256;
};

template <int HD>
__global__ void __launch_bounds__(kAttnThreads, 1)
    k_attn_bwd_dkdv(const __grid_constant__ CUtensorMap tk, const __grid_constant__ CUtensorMap tv,
                    const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tdo,
                    const BwdArgs a) {
  using C = DkdvCfg<HD>;
  constexpr int BN = C::BN, BM = C::BM;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sk = align1024(smem_raw);
  uint8_t* sv = sk + C::kKVBytes;
  uint8_t* sqd = sv + C::kKVBytes;  // stage s: Q at sqd + 2 s kQBytes, dO behind it
  float* svec = reinterpret_cast<float*>(sqd + kStages * 2 * C::kQBytes);  // stage s: lse2[BM], D[BM]
  uint64_t* kv_bar = reinterpret_cast<uint64_t*>(svec + kStages * 2 * BM);
  uint64_t* full = kv_bar + 1;
  uint64_t* empty = full + kStages;

  const int h = blockIdx.y, b = blockIdx.z, n0 = blockIdx.x * BN;
  const int q_lo = a.causal ? n0 / BM : 0, q_hi = (a.T + BM - 1) / BM;
  const int64_t bh = (int64_t)b * a.H + h, plane = (int64_t)gridDim.z * a.H * a.Tp;

  if (threadIdx.x == 0) {
    mbar_init(kv_bar, 1);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  bool ok = true;  // false: a barrier wait ran into the watchdog
  const int warp = threadIdx.x >> 5;
  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 256) {
      prefetch_tmap(&tk);
      prefetch_tmap(&tv);
      prefetch_tmap(&tq);
      prefetch_tmap(&tdo);
      mbar_expect_tx(kv_bar, 2 * C::kKVBytes);
      load_tile<HD, BN>(&tk, kv_bar, sk, n0, h, b);
      load_tile<HD, BN>(&tv, kv_bar, sv, n0, h, b);
      for (int qb = q_lo, it = 0; qb < q_hi; ++qb, ++it) {
        const int s = it % kStages;
        if (!(ok = mbar_wait_ok(&empty[s], ((it / kStages) & 1) ^ 1))) break;
        mbar_expect_tx(&full[s], 2 * C::kQBytes + 2 * C::kVecBytes);
        uint8_t* st = sqd + s * 2 * C::kQBytes;
        load_tile<HD, BM>(&tq, &full[s], st, qb * BM, h, b);
        load_tile<HD, BM>(&tdo, &full[s], st + C::kQBytes, qb * BM, h, b);
        const float* src = a.ws + bh * a.Tp + qb * BM;
        bulk_load(svec + s * 2 * BM, src, C::kVecBytes, &full[s]);
        bulk_load(svec + s * 2 * BM + BM, src + plane, C::kVecBytes, &full[s]);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const int j0 = n0 + wg * 64;                                // this warpgroup's key rows
    const int r0 = j0 + 16 * (t >> 5) + ((t & 31) >> 2);        // this thread's: r0, r0 + 8
    const int c0 = 2 * (t & 3);
    const float sl2 = a.scale_log2;
    float dk[HD / 2], dv[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dk[i] = dv[i] = 0.f;
    const uint32_t k_addr = smem_u32(sk), v_addr = smem_u32(sv);
    ok = mbar_wait_ok(kv_bar, 0);

    for (int qb = q_lo, it = 0; ok && qb < q_hi; ++qb, ++it) {
      const int s = it % kStages;
      const uint32_t q_addr = smem_u32(sqd + s * 2 * C::kQBytes), do_addr = q_addr + C::kQBytes;
      const float* lse2 = svec + s * 2 * BM;
      const float* dd = lse2 + BM;
      if (!(ok = mbar_wait_ok(&full[s], (it / kStages) & 1))) break;
      if (a.causal && qb * BM + BM - 1 < j0) {  // every query of the block precedes these keys
        if (t == 0) mbar_arrive(&empty[s]);
        continue;
      }
      float st[BM / 2];
      wgmma_fence();
      mma_ss<HD, BM, BN>(st, k_addr, wg * 64, q_addr);
      wgmma_commit();
      wgmma_wait<0>();

      const int q0 = qb * BM;
      const bool mask = a.causal && q0 < j0 + 63;
      uint32_t pt[BM / 4];
#pragma unroll
      for (int i = 0; i < BM / 2; i += 2) {
        const int col = 8 * (i >> 2) + c0, row = r0 + 8 * ((i >> 1) & 1);
        float p0 = exp2f(fmaf(st[i], sl2, -lse2[col])), p1 = exp2f(fmaf(st[i + 1], sl2, -lse2[col + 1]));
        if (mask) {
          if (q0 + col < row) p0 = 0.f;
          if (q0 + col + 1 < row) p1 = 0.f;
        }
        pt[i >> 1] = pack_bf16(p0, p1);
      }
      float dpt[BM / 2];
      wgmma_fence();
      mma_rs<HD, BM>(dv, pt, do_addr);
      wgmma_commit();
      mma_ss<HD, BM, BN>(dpt, v_addr, wg * 64, do_addr);
      wgmma_commit();
      wgmma_wait<0>();

      uint32_t ds[BM / 4];
#pragma unroll
      for (int i = 0; i < BM / 2; i += 2) {
        const int col = 8 * (i >> 2) + c0;
        const float2 pf = unpack_bf16(pt[i >> 1]);
        ds[i >> 1] = pack_bf16(pf.x * (dpt[i] - dd[col]), pf.y * (dpt[i + 1] - dd[col + 1]));
      }
      wgmma_fence();
      mma_rs<HD, BM>(dk, ds, q_addr);
      wgmma_commit();
      wgmma_wait<0>();
      if (t == 0) mbar_arrive(&empty[s]);
    }

    const float one[2] = {1.f, 1.f}, sc[2] = {a.scale, a.scale};
    store_rows<HD>(a.dv, a.dvs, b, h, r0, a.T, c0, dv, one);
    store_rows<HD>(a.dk, a.dks, b, h, r0, a.T, c0, dk, sc);
  }
  if (!ok) asm volatile("trap;");  // a protocol bug becomes a launch error, not a hung GPU
}

template <int HD> struct DqCfg {
  static constexpr int BM = 128, BN = 64;       // query rows per CTA, key rows per step
  static constexpr int kQBytes = BM * HD * 2;   // Q or dO
  static constexpr int kKVBytes = BN * HD * 2;  // K or V of one stage
  static constexpr int kSmemBytes = 2 * kQBytes + kStages * 2 * kKVBytes + 1024 + 256;
};

template <int HD>
__global__ void __launch_bounds__(kAttnThreads, 1)
    k_attn_bwd_dq(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tdo,
                  const __grid_constant__ CUtensorMap tk, const __grid_constant__ CUtensorMap tv,
                  const BwdArgs a) {
  using C = DqCfg<HD>;
  constexpr int BM = C::BM, BN = C::BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sq = align1024(smem_raw);
  uint8_t* sdo = sq + C::kQBytes;
  uint8_t* skv = sdo + C::kQBytes;  // stage s: K at skv + 2 s kKVBytes, V behind it
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(skv + kStages * 2 * C::kKVBytes);
  uint64_t* full = q_bar + 1;
  uint64_t* empty = full + kStages;

  const int m_blocks = (a.T + BM - 1) / BM;
  const int mb = a.causal ? m_blocks - 1 - (int)blockIdx.x : (int)blockIdx.x;
  const int h = blockIdx.y, b = blockIdx.z, m0 = mb * BM;
  const int n_all = (a.T + BN - 1) / BN;
  const int n_blocks = a.causal ? min(n_all, (m0 + BM) / BN) : n_all;

  if (threadIdx.x == 0) {
    mbar_init(q_bar, 1);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  bool ok = true;  // false: a barrier wait ran into the watchdog
  const int warp = threadIdx.x >> 5;
  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 256) {
      prefetch_tmap(&tq);
      prefetch_tmap(&tdo);
      prefetch_tmap(&tk);
      prefetch_tmap(&tv);
      mbar_expect_tx(q_bar, 2 * C::kQBytes);
      load_tile<HD, BM>(&tq, q_bar, sq, m0, h, b);
      load_tile<HD, BM>(&tdo, q_bar, sdo, m0, h, b);
      for (int n = 0; n < n_blocks; ++n) {
        const int s = n % kStages;
        if (!(ok = mbar_wait_ok(&empty[s], ((n / kStages) & 1) ^ 1))) break;
        mbar_expect_tx(&full[s], 2 * C::kKVBytes);
        uint8_t* st = skv + s * 2 * C::kKVBytes;
        load_tile<HD, BN>(&tk, &full[s], st, n * BN, h, b);
        load_tile<HD, BN>(&tv, &full[s], st + C::kKVBytes, n * BN, h, b);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const int r0 = m0 + wg * 64 + 16 * (t >> 5) + ((t & 31) >> 2);
    const int c0 = 2 * (t & 3);
    const float sl2 = a.scale_log2;
    const int64_t row_ws = ((int64_t)b * a.H + h) * a.Tp + r0, plane = (int64_t)gridDim.z * a.H * a.Tp;
    const float lse2[2] = {a.ws[row_ws], a.ws[row_ws + 8]};
    const float dd[2] = {a.ws[plane + row_ws], a.ws[plane + row_ws + 8]};
    float dq[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dq[i] = 0.f;
    const uint32_t q_addr = smem_u32(sq), do_addr = smem_u32(sdo);
    ok = mbar_wait_ok(q_bar, 0);

    for (int n = 0; ok && n < n_blocks; ++n) {
      const int s = n % kStages;
      const uint32_t k_addr = smem_u32(skv + s * 2 * C::kKVBytes), v_addr = k_addr + C::kKVBytes;
      if (!(ok = mbar_wait_ok(&full[s], (n / kStages) & 1))) break;
      if (a.causal && n * BN > m0 + wg * 64 + 63) {  // every key of the block follows these queries
        if (t == 0) mbar_arrive(&empty[s]);
        continue;
      }
      float sc[BN / 2], dp[BN / 2];
      wgmma_fence();
      mma_ss<HD, BN, BM>(sc, q_addr, wg * 64, k_addr);
      wgmma_commit();
      mma_ss<HD, BN, BM>(dp, do_addr, wg * 64, v_addr);
      wgmma_commit();
      wgmma_wait<0>();

      const int n0 = n * BN;
      const bool mask = (a.causal && n0 + BN - 1 > m0 + wg * 64) || n0 + BN > a.T;
      uint32_t ds[BN / 4];
#pragma unroll
      for (int i = 0; i < BN / 2; i += 2) {
        const int hh = (i >> 1) & 1, col = n0 + 8 * (i >> 2) + c0, row = r0 + 8 * hh;
        float p0 = exp2f(fmaf(sc[i], sl2, -lse2[hh])), p1 = exp2f(fmaf(sc[i + 1], sl2, -lse2[hh]));
        if (mask) {
          if (col >= a.T || (a.causal && col > row)) p0 = 0.f;
          if (col + 1 >= a.T || (a.causal && col + 1 > row)) p1 = 0.f;
        }
        const float2 pf = unpack_bf16(pack_bf16(p0, p1));
        ds[i >> 1] = pack_bf16(pf.x * (dp[i] - dd[hh]), pf.y * (dp[i + 1] - dd[hh]));
      }
      wgmma_fence();
      mma_rs<HD, BN>(dq, ds, k_addr);
      wgmma_commit();
      wgmma_wait<0>();
      if (t == 0) mbar_arrive(&empty[s]);
    }
    const float sc2[2] = {a.scale, a.scale};
    store_rows<HD>(a.dq, a.dqs, b, h, r0, a.T, c0, dq, sc2);
  }
  if (!ok) asm volatile("trap;");  // a protocol bug becomes a launch error, not a hung GPU
}

// ---- host side ---------------------------------------------------------------------------------------

// [B, H, T, hd] bf16 operand as a 4-D tensor map over (hd, T, H, B), boxes of 64 x box_rows.
int attn_tmap(CUtensorMap* map, const void* base, int64_t B, int64_t H, int64_t T, int64_t hd,
              const int64_t* st, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error(EDB_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[4] = {(cuuint64_t)hd, (cuuint64_t)T, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)st[2] * 2, (cuuint64_t)st[1] * 2, (cuuint64_t)st[0] * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult rc = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS)
    return set_error(EDB_E_CUDA, "attn: cuTensorMapEncodeTiled failed (%d)", (int)rc);
  return EDB_OK;
}

// Shapes and layouts every entry point needs: hd 64 or 128, a positive finite scale, 16-byte aligned
// pointers and positive 16-byte strides (TMA; no broadcast views), dims that fit the grid.  Returns EDB_OK, an error code, or -1 for an empty problem.
int attn_check(const char* who, int64_t B, int64_t H, int64_t T, int64_t hd, float scale,
               const void* const* ptrs, int n_ptrs, const int64_t* strides, int n_strides) {
  if (hd != 64 && hd != 128) return set_error(EDB_E_UNSUPPORTED, "%s: head dim %lld (64 or 128)", who, (long long)hd);
  // the online softmax shifts by the row maximum of the raw scores: right for scale > 0 only
  if (!(scale > 0.f) || !isfinite(scale))
    return set_error(EDB_E_UNSUPPORTED, "%s: scale %g (positive and finite)", who, (double)scale);
  if (B < 0 || H < 0 || T < 0 || strides == nullptr)
    return set_error(EDB_E_INVALID, "%s: B=%lld H=%lld T=%lld strides %p", who, (long long)B, (long long)H,
                     (long long)T, (const void*)strides);
  if (B == 0 || H == 0 || T == 0) return -1;
  if (B > 65535 || H > 65535 || T > (1 << 30))
    return set_error(EDB_E_UNSUPPORTED, "%s: B=%lld H=%lld T=%lld too large", who, (long long)B, (long long)H,
                     (long long)T);
  for (int i = 0; i < n_ptrs; ++i) {
    if (ptrs[i] == nullptr) return set_error(EDB_E_INVALID, "%s: null pointer %d", who, i);
    if ((uintptr_t)ptrs[i] & 15) return set_error(EDB_E_UNSUPPORTED, "%s: pointer %d not 16-byte aligned", who, i);
  }
  for (int i = 0; i < n_strides; ++i)
    if (strides[i] <= 0 || (strides[i] & 7) || strides[i] >= (1LL << 38))
      return set_error(EDB_E_UNSUPPORTED, "%s: stride %d = %lld (positive multiples of 8 elements)", who,
                       i, (long long)strides[i]);
  return EDB_OK;
}

template <typename K>
int set_smem(K kern, int bytes) {
  return cuda_check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes),
                    "attn: cudaFuncSetAttribute");
}

template <int HD>
int launch_fwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const FwdArgs& a,
               int B, int H, cudaStream_t s) {
  using C = FwdCfg<HD>;
  static int configured = set_smem(k_attn_fwd<HD>, C::kSmemBytes);
  if (configured != EDB_OK) return configured;
  k_attn_fwd<HD><<<dim3((a.T + C::BM - 1) / C::BM, H, B), kAttnThreads, C::kSmemBytes, s>>>(tq, tk, tv, a);
  count_launch();
  return cuda_check(cudaGetLastError(), "k_attn_fwd launch");
}

template <int HD>
int launch_bwd(const CUtensorMap* maps, const BwdArgs& a, int B, int H, cudaStream_t s) {
  using D1 = DkdvCfg<HD>;
  using D2 = DqCfg<HD>;
  static int configured = set_smem(k_attn_bwd_dkdv<HD>, D1::kSmemBytes) != EDB_OK
                              ? EDB_E_CUDA : set_smem(k_attn_bwd_dq<HD>, D2::kSmemBytes);
  if (configured != EDB_OK) return configured;
  const int64_t rows = (int64_t)B * H * a.Tp;
  k_attn_bwd_prep<HD><<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(a, rows);
  count_launch();
  EDB_CUDA(cudaGetLastError());
  // maps: k, v (128-row boxes), q, dO (64-row boxes) | q, dO (128-row boxes), k, v (64-row boxes)
  k_attn_bwd_dkdv<HD><<<dim3((a.T + D1::BN - 1) / D1::BN, H, B), kAttnThreads, D1::kSmemBytes, s>>>(
      maps[0], maps[1], maps[2], maps[3], a);
  count_launch();
  EDB_CUDA(cudaGetLastError());
  k_attn_bwd_dq<HD><<<dim3((a.T + D2::BM - 1) / D2::BM, H, B), kAttnThreads, D2::kSmemBytes, s>>>(
      maps[4], maps[5], maps[6], maps[7], a);
  count_launch();
  return cuda_check(cudaGetLastError(), "k_attn_bwd launch");
}

Rows rows_of(const int64_t* s) { return Rows{s[0], s[1], s[2]}; }

}  // namespace
}  // namespace edb

using namespace edb;

extern "C" {

int edb_attn_fwd(void* out, void* lse, const void* q, const void* k, const void* v, int64_t B, int64_t H,
                 int64_t T, int64_t hd, const int64_t* strides, float scale, int causal, void* stream) {
  const void* ptrs[4] = {q, k, v, out};
  int rc = attn_check("attn_fwd", B, H, T, hd, scale, ptrs, 4, strides, 12);
  if (rc < 0) return EDB_OK;
  if (rc != EDB_OK) return rc;
  if (lse == nullptr || ((uintptr_t)lse & 3) || strides[12] < 0 || strides[13] < 0 || strides[14] < 0)
    return set_error(EDB_E_INVALID, "attn_fwd: lse %p", lse);
  CUtensorMap tq, tk, tv;
  if ((rc = attn_tmap(&tq, q, B, H, T, hd, strides, 128)) != EDB_OK) return rc;
  if ((rc = attn_tmap(&tk, k, B, H, T, hd, strides + 3, 128)) != EDB_OK) return rc;
  if ((rc = attn_tmap(&tv, v, B, H, T, hd, strides + 6, 128)) != EDB_OK) return rc;
  FwdArgs a;
  a.o = static_cast<__nv_bfloat16*>(out);
  a.lse = static_cast<float*>(lse);
  a.os = rows_of(strides + 9);
  a.ls = rows_of(strides + 12);
  a.T = (int)T;
  a.causal = causal ? 1 : 0;
  a.scale_log2 = scale * kLog2e;
  cudaStream_t s = (cudaStream_t)stream;
  return hd == 64 ? launch_fwd<64>(tq, tk, tv, a, (int)B, (int)H, s)
                  : launch_fwd<128>(tq, tk, tv, a, (int)B, (int)H, s);
}

int edb_attn_bwd_workspace(int64_t B, int64_t H, int64_t T, size_t* bytes) {
  if (B < 0 || H < 0 || T < 0 || bytes == nullptr) return set_error(EDB_E_INVALID, "attn_bwd_workspace");
  *bytes = (size_t)(2 * B * H * ((T + kPad - 1) / kPad * kPad) * 4);
  return EDB_OK;
}

int edb_attn_bwd(void* dq, void* dk, void* dv, const void* dout, const void* q, const void* k,
                 const void* v, const void* out, const void* lse, void* workspace, int64_t B, int64_t H,
                 int64_t T, int64_t hd, const int64_t* strides, float scale, int causal, void* stream) {
  const void* ptrs[9] = {dout, q, k, v, out, dq, dk, dv, workspace};
  int rc = attn_check("attn_bwd", B, H, T, hd, scale, ptrs, 9, strides, 24);
  if (rc < 0) return EDB_OK;
  if (rc != EDB_OK) return rc;
  if (lse == nullptr || ((uintptr_t)lse & 3) || strides[24] < 0 || strides[25] < 0 || strides[26] < 0)
    return set_error(EDB_E_INVALID, "attn_bwd: lse %p", lse);
  CUtensorMap maps[8];
  const void* srcs[8] = {k, v, q, dout, q, dout, k, v};
  const int64_t* sts[8] = {strides + 6, strides + 9, strides + 3, strides, strides + 3, strides, strides + 6,
                           strides + 9};
  const int boxes[8] = {128, 128, 64, 64, 128, 128, 64, 64};
  for (int i = 0; i < 8; ++i)
    if ((rc = attn_tmap(&maps[i], srcs[i], B, H, T, hd, sts[i], boxes[i])) != EDB_OK) return rc;
  BwdArgs a;
  a.dq = static_cast<__nv_bfloat16*>(dq);
  a.dk = static_cast<__nv_bfloat16*>(dk);
  a.dv = static_cast<__nv_bfloat16*>(dv);
  a.dout = static_cast<const __nv_bfloat16*>(dout);
  a.out = static_cast<const __nv_bfloat16*>(out);
  a.lse = static_cast<const float*>(lse);
  a.ws = static_cast<float*>(workspace);
  a.dos = rows_of(strides);
  a.outs = rows_of(strides + 12);
  a.dqs = rows_of(strides + 15);
  a.dks = rows_of(strides + 18);
  a.dvs = rows_of(strides + 21);
  a.ls = rows_of(strides + 24);
  a.T = (int)T;
  a.Tp = (int)((T + kPad - 1) / kPad * kPad);
  a.H = (int)H;
  a.causal = causal ? 1 : 0;
  a.scale = scale;
  a.scale_log2 = scale * kLog2e;
  cudaStream_t s = (cudaStream_t)stream;
  return hd == 64 ? launch_bwd<64>(maps, a, (int)B, (int)H, s) : launch_bwd<128>(maps, a, (int)B, (int)H, s);
}

}  // extern "C"
