// Dense bf16 GEMM on Hopper tensor cores (wgmma + TMA + mbarrier), the compute half of the
// sharded-op kernel dispatch: the aten.mm.default nodes of the sharded FX graph
// (Linear fwd / dgrad / wgrad; SURVEY.md §8 a14) land here.
//
//   C[M,N] (bf16) = A · B, fp32 accumulation in registers.
//     A: K-major  ([M,K] row-major)  or MN-major (stored [K,M])
//     B: K-major  ([N,K] row-major, i.e. nn.Linear weight) or MN-major (stored [K,N])
//
// Structure (one persistent CTA per SM, 288 threads):
//   warps 0..7 : two consumer warpgroups — each issues wgmma.mma_async (64 x BN x 16) on its 64
//                rows of the 128 x BN tile with the accumulator in registers, then runs the
//                epilogue: registers -> bf16 -> 128B-swizzled smem -> TMA store
//   warp 8     : TMA producer — one lane issues cp.async.bulk.tensor tiles of A and B into a
//                4/6-stage smem ring, already loading the next tile while the consumers run the
//                epilogue
// Synchronisation is mbarrier-only (full/empty per smem stage).
//
// Shared-memory tiles use the canonical 128-byte-swizzle wgmma layouts, written by TMA with
// CU_TENSOR_MAP_SWIZZLE_128B and described to the tensor core with matching smem descriptors
// (K-major: SBO = 1024 B; MN-major: one 64-element atom per TMA box, LBO = atom stride).
#include <cuda.h>
#include <cuda_bf16.h>

#include "edb_internal.cuh"

namespace edb {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 bytes = one swizzle atom
constexpr int MMA_K = 16;
constexpr int kConsumerThreads = 256;                 // two warpgroups, 64 tile rows each
constexpr int kGemmThreads = kConsumerThreads + 32;   // + the producer warp
constexpr int kSmemABytes = BM * BK * 2;  // 16 KiB

// A 128 x 256 tile reads 48 KiB of operands per 64-deep k-block for 2 x 64 x 256 x 64 MMAs, a
// 128 x 128 tile 32 KiB for half the work: 256 wide whenever N allows.  Stages fill the 227 KiB an
// H100 block may use (4 x 48 KiB or 6 x 32 KiB, + 32 KiB of epilogue staging).
template <int BN> struct TileCfg {
  static constexpr int kSmemBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kSmemABytes + kSmemBBytes;
  static constexpr int kStages = (BN == 256) ? 4 : 6;
  static constexpr int kEpiBufBytes = BM * 64 * 2;  // one 128 x 64 bf16 store box (128B swizzle)
  static constexpr int kEpiBufs = 2;
  static constexpr int kSmemBytes =
      kStages * kStageBytes + kEpiBufs * kEpiBufBytes + 1024 /*align*/ + 256 /*barriers*/;
};

// ---- PTX wrappers ------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t addr, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(addr), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin on an mbarrier phase.  A watchdog turns a protocol bug into a trap (kernel error) instead
// of a hung GPU: 4 s is ~1000x the longest legitimate wait of any role in these kernels.
// No printf: it is a function call, and ptxas serialises the wgmmas of a kernel whose wgmma
// pipeline may cross one.  The trap surfaces as a launch error on the host.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  if (mbar_try_wait(addr, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(addr, parity)) {
    if ((++spins & 0xfff) == 0 && globaltimer_ns() - t0 > 4000000000ull) {
      asm volatile("trap;");
    }
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* smem,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];" ::"r"(smem_u32(smem)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem, int c0,
                                             int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map),
      "r"(smem_u32(smem)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N> __device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void epi_bar_sync() {
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N> __device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x N] (+)= A[64 x 16] · B[16 x N]; TA / TB = 1: operand stored MN-major (transposed).
// scale_d == 0 starts a fresh accumulator.  The accumulator fragment of thread t of the warpgroup:
// d[i] = D[16 (t / 32) + (t % 32) / 4 + 8 ((i / 2) % 2)][8 (i / 4) + 2 (t % 4) + i % 2].
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float* d, uint64_t desc_a, uint64_t desc_b,
                                                  uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, %67, %68;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float* d, uint64_t desc_a, uint64_t desc_b,
                                                  uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, %131, %132;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}

// ---- descriptors -------------------------------------------------------------------------------------

// wgmma shared-memory matrix descriptor:
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4
//   [49,52) base offset = 0 (tiles are 1024-byte aligned)   [62,64) layout type: 1 = SWIZZLE_128B
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes,
                                                   uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

struct GemmParams {
  __nv_bfloat16* C;
  const __nv_bfloat16* bias;  // optional [N] row vector added in the epilogue (aten.addmm)
  int64_t ldc;
  int M, N, K;
  int m_tiles, n_tiles;
  // split-K (MODE_PLAIN only): work unit = (tile, k-slice); every slice writes its fp32 partial
  // tile to `partial` [splits][M][ldp] and k_splitk_reduce sums the slices in a fixed order
  int splits, kb_per_split;
  float* partial;
  int64_t ldp;
  // push mode (MODE_PLAIN, edb_gemm_push_bf16): row block m of C belongs to group member
  // m / push_mtc and is TMA-stored into that member's receive slot (store map cm.m[owner]) instead
  // of C; m_rot rotates the m order so that the ranks do not all push to the same owner at once
  int push_n, push_mtc, m_rot;
  // how a pushing CTA retires: 2 = wait for the completion of its TMA stores + system-scope fence,
  // 1 = completion only, 0 = only until the staging smem has been read (grid completion then
  // covers the stores, as it does for every ordinary TMA-store epilogue)
  int push_sync;
  // fused elementwise epilogue with a second operand `aux` [M, N] bf16 (row stride ld_aux):
  //   EPI_ADD      C = bf16(acc + bias + aux)                  (residual add behind a Linear)
  //   EPI_GELU_BWD C = bf16(acc * gelu'(aux)), tanh approximation, ATen's formula in fp32
  //                (aten.gelu_backward(grad = this GEMM, self = aux): the dgrad GEMM of the MLP's
  //                second Linear produces d(pre-activation) directly)
  const __nv_bfloat16* aux;
  int64_t ld_aux;
  int epi_op;
};
enum { EPI_NONE = 0, EPI_ADD = 1, EPI_GELU_BWD = 2 };

__device__ __forceinline__ float gelu_tanh_grad(float x) {
  // at::native GeluBackwardCUDAKernelImpl, approximate == 'tanh' (opmath = float)
  const float kBeta = 0.7978845608028654f;  // sqrt(2) * (2/sqrt(pi)) * 0.5
  const float kKappa = 0.044715f;
  const float x_sq = x * x;
  const float inner = kBeta * (x + kKappa * x_sq * x);
  // tanh and sech^2 from ONE exponential: e = exp(-2|u|) (ex2.approx, rel. error 2^-22),
  // tanh = sign(u)(1-e)/(1+e), 1 - tanh^2 = 4e/(1+e)^2.  (tanh.approx.f32 is one MUFU op cheaper but
  // its 2^-11 error is absolute near saturation: 1 - t*t then loses everything for |x| > 3 and the
  // gradient of a saturated unit came out as ~3 % of dy instead of ~0.  tanhf costs more than the
  // main loop: 16.7 M evaluations per MLP dgrad GEMM sit on the four epilogue warps.)
  const float au = fabsf(inner);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-2.885390081777927f * au));  // 2 / ln 2
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  const float t = copysignf((1.0f - e) * r, inner);
  const float tanh_d = 4.0f * e * r * r;
  const float left = 0.5f * x, right = 1.0f + t;
  const float left_d = 0.5f * right;
  const float inner_d = kBeta * (1.0f + 3.0f * kKappa * x_sq);
  return left_d + left * tanh_d * inner_d;
}

// Fusion modes of the GEMM kernel
//   MODE_PLAIN : C = A.B
//   MODE_AG    : B (weights, [N,K] K-major) is sharded S(0) over the group; a few "comm" CTAs pull the
//                peer shards over NVLink with TMA bulk copies into the local gathered buffer while
//                the MMA CTAs start on the local shard and pick up chunks as their flags arrive
//                (all_gather_end -> aten.mm of the sharded graph in one kernel)
//   MODE_RS    : the partial product C is reduce-scattered over its rows: the epilogue TMA-stores
//                every tile straight into the owner's receive slot over NVLink (own rows last),
//                per-chunk flags tell the owner when a source is complete, and the tail of the same
//                kernel reduces the n slots in rank order with scale + cast
//                (aten.mm -> reduce_scatter_start in one kernel)
enum { MODE_PLAIN = 0, MODE_AG = 1, MODE_RS = 2 };
constexpr int kMaxPfItems = 4;
constexpr int kPfSlots = 12, kPfDepth = 8;  // 16 KiB slots of the prefetch ring / loads in flight
constexpr int F_TILECNT = 96;  // flag-block words [96,104): per-chunk completion counters

struct FusedArgs {
  FlagCtx f;
  int n_comm;  // MODE_AG: number of comm CTAs at the end of the grid
  // MODE_AG
  const char* shard_src[kMaxGroup];  // member p's shard (peer mapped); [me] is local
  char* full_dst;                    // local gathered buffer
  int64_t shard_bytes;
  int ag_rows;        // rows of B per shard (N / n)
  int ag_first_tile;  // n-tile containing the first row of my shard
  // MODE_RS
  char* recv_base;      // my receive buffer: n slots of chunk_bytes
  int64_t chunk_bytes;  // (M/n) * N * 2
  void* rs_dst;
  float rs_scale;
  int rs_out_dtype;
  int tiles_per_chunk;
  // deferred reduce-scatter: the kernel only pushes its tiles (flag words F_CHUNK + 8 + src) and
  // records its op number in rs_state[0]; k_rs_finish reduces the slots later (rs_state[1] = the op
  // number of that reduction, which guards the slots against the next step's pushes)
  int rs_defer;
  uint64_t* rs_state;
  // epoch mode (edb_ag_gemm_epoch_bf16): no handshake with the peers inside the kernel — an
  // edb_epoch_barrier earlier on the stream made every member's shard final, and the next barrier
  // comes before anybody overwrites it.  Only the local chunk flags (comm CTAs -> MMA CTAs) remain.
  int epoch;
  // all-gather PREFETCH riding on a plain GEMM (edb_gemm_pf_bf16): the first pf_ctas CTAs of the
  // grid do no MMA work; they copy, for each item and each group member p, the byte range
  // [src_off, src_off + bytes) of p's symmetric heap into local dst_off + p * dst_stride — the
  // operand of a LATER kernel (next layer's weight), so nobody in this kernel waits for the data
  // and the consumer is an ordinary GEMM.  Epoch protocol: the sources are final since the last
  // edb_epoch_barrier.
  int pf_ctas, pf_items, pf_n;
  const char* pf_heap[kMaxGroup];  // members' heaps (peer mapped), [pf_me] = local
  char* pf_local;
  uint64_t pf_src[kMaxPfItems], pf_dst[kMaxPfItems];
  int64_t pf_bytes[kMaxPfItems], pf_stride[kMaxPfItems];
  // pf_sstride: member p's source is at pf_src + p * pf_sstride (0: the same offset everywhere).
  // With pf_sstride == pf_stride and pf_src == pf_dst every member's shard LIVES in its slot of
  // the gathered buffer: nothing to copy for the own range (pf_inplace), n-1 remote ranges only.
  int64_t pf_sstride[kMaxPfItems];
  int pf_inplace[kMaxPfItems];
};
constexpr int F_PUSHED = F_CHUNK + 8;  // [40..47] PUSHED[p]: peer p's deferred-RS tiles of op q landed

struct CMaps {
  CUtensorMap m[kMaxGroup];  // MODE_RS: store map of member p's receive slot [me]; MODE_AG: m[0] = local shard
};

template <int MODE>
__device__ __forceinline__ void tile_coords(int t, const GemmParams& p, const FusedArgs& fa,
                                            int& m_blk, int& n_blk, int& chunk) {
  if (MODE == MODE_AG) {
    // n-tiles in rotated order starting at the tile that holds my own shard (needs no transfer),
    // then in the order the comm CTAs pull the peers' shards
    const int ni = t / p.m_tiles;
    n_blk = (fa.ag_first_tile + ni) % p.n_tiles;
    m_blk = t - ni * p.m_tiles;
    chunk = -1;  // a tile may span several shards: see the producer
  } else if (MODE == MODE_RS) {
    const int mtc = p.m_tiles / fa.f.n;  // m-tiles per chunk
    const int tpc = mtc * p.n_tiles;
    const int ci = t / tpc, w = t - ci * tpc;
    chunk = (fa.f.me + 1 + ci) % fa.f.n;  // own rows last: their reduction needs the peers anyway
    m_blk = chunk * mtc + w % mtc;
    n_blk = w / mtc;
  } else {
    chunk = 0;
    m_blk = (t % p.m_tiles + p.m_rot) % p.m_tiles;
    n_blk = t / p.m_tiles;
  }
}

__device__ __forceinline__ void bulk_load(void* smem, const void* gsrc, uint32_t bytes,
                                          uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void bulk_store(void* gdst, const void* smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"(smem_u32(smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() {
  asm volatile("fence.proxy.async;" ::: "memory");
}
__device__ __forceinline__ void spin_wait_gpu(const uint64_t* flag, uint64_t target) {
  if (ld_acquire_gpu(flag) >= target) return;
  const uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (ld_acquire_gpu(flag) < target) {
    __nanosleep(32);
    if ((++spins & 0xfff) == 0 && globaltimer_ns() - t0 > 4000000000ull) asm volatile("trap;");
  }
}

// Prefetch CTA (see FusedArgs::pf_*): one thread drives a TMA bulk-copy ring peer HBM -> smem ->
// local HBM over the 16 KiB blocks of all (item, member) ranges; block b belongs to CTA
// b % pf_ctas, so the CTAs stream neighbouring blocks and every range finishes at about the same
// time.  No flags: the consumer is a later kernel on the stream.
__device__ __forceinline__ void pf_role(const FusedArgs& fa, uint8_t* smem, int idx, int nctas) {
  constexpr int S = kPfSlots, D = kPfDepth, SLOT = 16384;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * SLOT);
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) mbar_init(&full[s], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  // flat block numbering: item-major, member-major inside an item, remote members first
  uint32_t n_load = 0, n_store = 0;
  struct Cur { int it, k; int64_t blk; };
  auto advance = [&](Cur& c) {
    // move to the next block owned by this CTA; returns false at the end
    while (c.it < fa.pf_items) {
      const int64_t nblk = (fa.pf_bytes[c.it] + SLOT - 1) / SLOT;
      const int members = fa.pf_inplace[c.it] ? fa.pf_n - 1 : fa.pf_n;  // own range last / skipped
      if (c.k < members && c.blk < nblk) return true;
      if (c.k < members) c.blk -= nblk;  // keep the round-robin phase across ranges
      if (++c.k >= members) {
        c.k = 0;
        ++c.it;
      }
    }
    return false;
  };
  Cur ld = {0, 0, (int64_t)idx}, stc = {0, 0, (int64_t)idx};
  bool more = advance(ld);
  int inflight = 0;
  while (more || inflight > 0) {
    if (more && inflight < D) {
      const uint32_t slot = n_load % S;
      if (n_load >= (uint32_t)S) tma_store_wait_read<S - D - 1>();
      const int p = (fa.f.me + 1 + ld.k) % fa.pf_n;  // own range last (a local copy)
      const int64_t off = ld.blk * SLOT;
      const int64_t left = fa.pf_bytes[ld.it] - off;
      const uint32_t bytes = (uint32_t)(left < SLOT ? left : SLOT);
      mbar_expect_tx(&full[slot], bytes);
      bulk_load(smem + slot * SLOT,
                fa.pf_heap[p] + fa.pf_src[ld.it] + (int64_t)p * fa.pf_sstride[ld.it] + off, bytes,
                &full[slot]);
      ++n_load;
      ++inflight;
      ld.blk += nctas;
      more = advance(ld);
      continue;
    }
    // oldest load -> store
    advance(stc);
    const uint32_t slot = n_store % S;
    mbar_wait(&full[slot], (n_store / S) & 1);
    const int p = (fa.f.me + 1 + stc.k) % fa.pf_n;
    const int64_t off = stc.blk * SLOT;
    const int64_t left = fa.pf_bytes[stc.it] - off;
    const uint32_t bytes = (uint32_t)(left < SLOT ? left : SLOT);
    bulk_store(fa.pf_local + fa.pf_dst[stc.it] + (int64_t)p * fa.pf_stride[stc.it] + off,
               smem + slot * SLOT, bytes);
    tma_store_commit();
    ++n_store;
    --inflight;
    stc.blk += nctas;
  }
  tma_store_wait_all();
}

__global__ void __launch_bounds__(32, 1) k_ag_prefetch(const __grid_constant__ FusedArgs fa) {
  extern __shared__ uint8_t pf_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(pf_smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  pf_role(fa, smem, (int)blockIdx.x, (int)gridDim.x);
}

// Epoch-mode comm CTA: the same TMA bulk-copy ring, but ONE software pipeline over the blocks of
// all shards — no drain between shards (the per-op variant below pays a load + store latency per
// shard, ~4 us x (n-1) at n = 8) and no flag traffic with the peers at all.  A shard is announced
// to the MMA CTAs once `wait_group` proves its last store complete, which lags kLag stores behind.
__device__ __forceinline__ void ag_comm_role_epoch(const FusedArgs& fa, uint8_t* smem, int comm_idx,
                                                   uint64_t q) {
  constexpr int S = 8, D = 5, SLOT = 16384, kLag = 2;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * SLOT);
  const FlagCtx& f = fa.f;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) mbar_init(&full[s], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int64_t per = ((fa.shard_bytes + fa.n_comm - 1) / fa.n_comm + SLOT - 1) / SLOT * SLOT;
  const int64_t lo = (int64_t)comm_idx * per;
  const int64_t hi = lo + per < fa.shard_bytes ? lo + per : fa.shard_bytes;
  const int nblk = hi > lo ? (int)((hi - lo + SLOT - 1) / SLOT) : 0;
  const int total = nblk * f.n;
  auto announce = [&](int k) {
    const int c = (f.me + k) % f.n;
    const unsigned long long prev =
        atomicAdd(reinterpret_cast<unsigned long long*>(f.local + F_AGTILE + c), 1ULL);
    if (prev == (unsigned long long)fa.n_comm - 1) {
      f.local[F_AGTILE + c] = 0;
      __threadfence();
      st_release_gpu(f.local + F_AGCHUNK + c, q);
    }
  };
  if (nblk == 0) {
    for (int k = 0; k < f.n; ++k) announce(k);  // nothing to move for this CTA: still counted
  } else {
    uint32_t n_load = 0, n_store = 0;
    int next_announce = 0;  // shards [0, next_announce) have been announced
    for (int g = 0; g < total + D; ++g) {
      if (g < total) {
        const int k = g / nblk, i = g - k * nblk;
        const int c = (f.me + k) % f.n;
        const uint32_t slot = n_load % S;
        if (n_load >= (uint32_t)S) tma_store_wait_read<S - D - 1>();
        const int64_t left = hi - lo - (int64_t)i * SLOT;
        const uint32_t bytes = (uint32_t)(left < SLOT ? left : SLOT);
        mbar_expect_tx(&full[slot], bytes);
        bulk_load(smem + slot * SLOT, fa.shard_src[c] + lo + (int64_t)i * SLOT, bytes, &full[slot]);
        ++n_load;
      }
      if (g >= D) {
        const int j = g - D;
        const int k = j / nblk, i = j - k * nblk;
        const int c = (f.me + k) % f.n;
        const uint32_t slot = n_store % S;
        mbar_wait(&full[slot], (n_store / S) & 1);
        const int64_t left = hi - lo - (int64_t)i * SLOT;
        const uint32_t bytes = (uint32_t)(left < SLOT ? left : SLOT);
        bulk_store(fa.full_dst + (int64_t)c * fa.shard_bytes + lo + (int64_t)i * SLOT,
                   smem + slot * SLOT, bytes);
        tma_store_commit();
        ++n_store;
        // shard `next_announce` ended with store number (next_announce + 1) * nblk: once kLag more
        // stores have been committed, wait_group<kLag> proves it complete
        if ((int)n_store - kLag >= (next_announce + 1) * nblk) {
          asm volatile("cp.async.bulk.wait_group %0;" ::"n"(kLag) : "memory");
          fence_proxy_async_all();
          __threadfence();
          while ((int)n_store - kLag >= (next_announce + 1) * nblk) announce(next_announce++);
        }
      }
    }
    tma_store_wait_all();
    fence_proxy_async_all();
    __threadfence();
    while (next_announce < f.n) announce(next_announce++);
  }
  // advance the launch number once every CTA of this launch has read the old one
  const unsigned long long prev =
      atomicAdd(reinterpret_cast<unsigned long long*>(f.local + F_AGDONE), 1ULL);
  if (prev == (unsigned long long)fa.n_comm - 1) {
    f.local[F_AGDONE] = 0;
    while (ld_acquire_gpu(f.local + F_AGCNT) < (uint64_t)gridDim.x) __nanosleep(64);
    f.local[F_AGCNT] = 0;
    st_release_gpu(f.local + F_AGSEQ, q);
  }
}

// MODE_AG comm CTA: one thread drives a TMA bulk-copy ring  peer HBM -> smem -> local HBM.
__device__ __forceinline__ void ag_comm_role(const FusedArgs& fa, uint8_t* smem, int comm_idx,
                                             uint64_t q) {
  constexpr int S = 8, D = 4, SLOT = 16384;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * SLOT);
  const FlagCtx& f = fa.f;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) mbar_init(&full[s], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int w_chunk = F_CHUNK, w_tile = F_TILECNT;
  if (comm_idx == 0) {
    // my shard was written by earlier kernels of this stream: publish it
    __threadfence_system();
    for (int pidx = 0; pidx < f.n; ++pidx)
      if (pidx != f.me) st_release_sys(f.peer[pidx] + F_READY + f.me, q);
  }
  uint32_t n_load = 0, n_store = 0;
  const int64_t per = ((fa.shard_bytes + fa.n_comm - 1) / fa.n_comm + SLOT - 1) / SLOT * SLOT;
  const int64_t lo = (int64_t)comm_idx * per;
  const int64_t hi = lo + per < fa.shard_bytes ? lo + per : fa.shard_bytes;
  const int64_t nblk = hi > lo ? (hi - lo + SLOT - 1) / SLOT : 0;
  for (int k = 0; k < f.n; ++k) {
    const int c = (f.me + k) % f.n;
    if (c != f.me) spin_wait_sys(f.local + F_READY + c, q, f.timeout_ns, f.local + F_ERR);
    const char* src = fa.shard_src[c] + lo;
    char* dst = fa.full_dst + (int64_t)c * fa.shard_bytes + lo;
    for (int64_t i = 0; i < nblk + D; ++i) {
      if (i < nblk) {
        const uint32_t slot = n_load % S;
        if (n_load >= (uint32_t)S) tma_store_wait_read<S - D - 1>();
        const int64_t left = hi - lo - i * SLOT;
        const uint32_t bytes = (uint32_t)(left < SLOT ? left : SLOT);
        mbar_expect_tx(&full[slot], bytes);
        bulk_load(smem + slot * SLOT, src + i * SLOT, bytes, &full[slot]);
        ++n_load;
      }
      if (i >= D) {
        const int64_t j = i - D;
        const uint32_t slot = n_store % S;
        mbar_wait(&full[slot], (n_store / S) & 1);
        const int64_t left = hi - lo - j * SLOT;
        const uint32_t bytes = (uint32_t)(left < SLOT ? left : SLOT);
        bulk_store(dst + j * SLOT, smem + slot * SLOT, bytes);
        tma_store_commit();
        ++n_store;
      }
    }
    tma_store_wait_all();
    fence_proxy_async_all();
    __threadfence();
    const unsigned long long prev =
        atomicAdd(reinterpret_cast<unsigned long long*>(f.local + w_tile + c), 1ULL);
    if (prev == (unsigned long long)fa.n_comm - 1) {
      f.local[w_tile + c] = 0;
      __threadfence();
      st_release_gpu(f.local + w_chunk + c, q);
    }
  }
  // end of the op: DONE to the peers, SEQ locally — but only after every CTA of this launch has
  // read the old SEQ (slow starters would otherwise compute the wrong op number)
  const unsigned long long prev =
      atomicAdd(reinterpret_cast<unsigned long long*>(f.local + F_CNT_B), 1ULL);
  if (prev == (unsigned long long)fa.n_comm - 1) {
    f.local[F_CNT_B] = 0;
    while (ld_acquire_gpu(f.local + F_CNT_C) < (uint64_t)gridDim.x) __nanosleep(64);
    f.local[F_CNT_C] = 0;
    __threadfence_system();
    for (int pidx = 0; pidx < f.n; ++pidx)
      if (pidx != f.me) st_release_sys(f.peer[pidx] + F_DONE + f.me, q);
    st_release_gpu(f.local + F_SEQ, q);
  }
}

template <typename Out>
__device__ __forceinline__ void rs_store(Out* out, int64_t i, const float* acc) {
  if (sizeof(Out) == 4) {
    float4* o = reinterpret_cast<float4*>(out) + 2 * i;
    o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  } else {
    uint4 o;
    __nv_bfloat162 h0 = __floats2bfloat162_rn(acc[0], acc[1]);
    __nv_bfloat162 h1 = __floats2bfloat162_rn(acc[2], acc[3]);
    __nv_bfloat162 h2 = __floats2bfloat162_rn(acc[4], acc[5]);
    __nv_bfloat162 h3 = __floats2bfloat162_rn(acc[6], acc[7]);
    o.x = *reinterpret_cast<uint32_t*>(&h0);
    o.y = *reinterpret_cast<uint32_t*>(&h1);
    o.z = *reinterpret_cast<uint32_t*>(&h2);
    o.w = *reinterpret_cast<uint32_t*>(&h3);
    reinterpret_cast<uint4*>(out)[i] = o;
  }
}

// Sum the n receive slots in rank order (fp32), scale, cast.  All slots are local memory; every
// load of an iteration is issued before the first add so that n x U 16-byte loads are in flight.
template <typename Out>
__device__ __forceinline__ void rs_tail_reduce(const FusedArgs& fa, uint64_t tid, uint64_t nthr) {
  const int64_t nvec = fa.chunk_bytes / 16;  // 8 bf16 per vector
  const int n = fa.f.n;
  Out* out = static_cast<Out*>(fa.rs_dst);
  constexpr int U = 2;
  for (int64_t i0 = tid; i0 < nvec; i0 += U * nthr) {
    uint4 raw[U][kMaxGroup];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * (int64_t)nthr;
      if (i < nvec) {
#pragma unroll
        for (int s = 0; s < kMaxGroup; ++s)
          if (s < n)
            raw[u][s] = *reinterpret_cast<const uint4*>(fa.recv_base + (int64_t)s * fa.chunk_bytes + i * 16);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * (int64_t)nthr;
      if (i >= nvec) break;
      float acc[8];
#pragma unroll
      for (int s = 0; s < kMaxGroup; ++s) {
        if (s < n) {
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[u][s]);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 v = __bfloat1622float2(h[e]);
            if (s == 0) {
              acc[2 * e] = v.x;
              acc[2 * e + 1] = v.y;
            } else {
              acc[2 * e] += v.x;
              acc[2 * e + 1] += v.y;
            }
          }
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] *= fa.rs_scale;
      rs_store<Out>(out, i, acc);
    }
  }
}

// ---- kernel ------------------------------------------------------------------------------------------

// One consumer warpgroup's accumulator: rows 64 wg + [0, 64) of the tile, all BN columns.
// Epilogue helpers below address it through the fragment layout of wgmma_m64n*k16.
template <int BN, bool A_KMAJOR, bool B_KMAJOR>
__device__ __forceinline__ void mma_k_block(float* acc, uint32_t a_addr, uint32_t b_addr, bool fresh) {
#pragma unroll
  for (int k = 0; k < BK / MMA_K; ++k) {
    // K-major: the 16-element k step moves 32 bytes inside the 128-byte swizzle row;
    // MN-major: it moves 16 k rows of 128 bytes
    const uint64_t da = A_KMAJOR ? make_smem_desc(a_addr + k * MMA_K * 2, 16, 1024)
                                 : make_smem_desc(a_addr + k * MMA_K * 128, 64 * BK * 2, 1024);
    const uint64_t db = B_KMAJOR ? make_smem_desc(b_addr + k * MMA_K * 2, 16, 1024)
                                 : make_smem_desc(b_addr + k * MMA_K * 128, 64 * BK * 2, 1024);
    const uint32_t scale_d = (fresh && k == 0) ? 0u : 1u;
    if (BN == 256) wgmma_m64n256k16<A_KMAJOR ? 0 : 1, B_KMAJOR ? 0 : 1>(acc, da, db, scale_d);
    else wgmma_m64n128k16<A_KMAJOR ? 0 : 1, B_KMAJOR ? 0 : 1>(acc, da, db, scale_d);
  }
}

template <int BN, bool A_KMAJOR, bool B_KMAJOR, int MODE>
__global__ void __launch_bounds__(kGemmThreads, 1)
    k_gemm_bf16(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const __grid_constant__ CUtensorMap tmap_c, const GemmParams p,
                const __grid_constant__ FusedArgs fa, const __grid_constant__ CMaps cm) {
  using Cfg = TileCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  __shared__ uint64_t s_q;
  __shared__ int s_last;
  uint64_t q = 0;
  const int n_gemm_ctas = (MODE == MODE_AG) ? (int)gridDim.x - fa.n_comm
                                             : (MODE == MODE_PLAIN ? (int)gridDim.x - fa.pf_ctas : (int)gridDim.x);

  if (MODE == MODE_RS) {
    if (fa.rs_defer) {
      // no lockstep with the peers: the receive slots belong to this weight alone, and the owners
      // finished reducing their previous content in op rs_state[1] (same op number on every rank)
      if (threadIdx.x == 0) s_q = ld_relaxed_gpu(fa.f.local + F_SEQ) + 1;
      if ((int)threadIdx.x < fa.f.n && (int)threadIdx.x != fa.f.me) {
        const uint64_t prev = ld_relaxed_gpu(fa.rs_state + 1);
        if (prev) spin_wait_sys(fa.f.local + F_DONE + threadIdx.x, prev, fa.f.timeout_ns, fa.f.local + F_ERR);
      }
      __syncthreads();
      q = s_q;
    } else {
      q = begin_op(fa.f, &s_q);  // WAR guard: peers are done with my buffers of earlier ops
    }
  } else if (MODE == MODE_AG) {
    if (threadIdx.x == 0) {
      s_q = ld_relaxed_gpu(fa.f.local + (fa.epoch ? F_AGSEQ : F_SEQ)) + 1;
      atomicAdd(reinterpret_cast<unsigned long long*>(fa.f.local + (fa.epoch ? F_AGCNT : F_CNT_C)), 1ULL);
    }
    __syncthreads();
    q = s_q;
    // the comm CTAs are the producers the MMA CTAs spin on: they get the LOWEST block indices so
    // that they are scheduled first even when the grid is not fully co-resident
    if ((int)blockIdx.x < fa.n_comm) {
      if (fa.epoch) ag_comm_role_epoch(fa, smem, (int)blockIdx.x, q);
      else ag_comm_role(fa, smem, (int)blockIdx.x, q);
      return;
    }
  }
  if (MODE == MODE_PLAIN && fa.pf_ctas > 0 && (int)blockIdx.x < fa.pf_ctas) {
    // prefetch CTAs: lowest block indices, no part in the GEMM
    pf_role(fa, smem, (int)blockIdx.x, fa.pf_ctas);
    return;
  }
  const int cta = (MODE == MODE_AG) ? (int)blockIdx.x - fa.n_comm
                                    : (MODE == MODE_PLAIN ? (int)blockIdx.x - fa.pf_ctas : (int)blockIdx.x);

  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kSmemABytes;
  uint8_t* smem_epi = smem + kStages * Cfg::kStageBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_epi + Cfg::kEpiBufs * Cfg::kEpiBufBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int k_blocks = (p.K + BK - 1) / BK;
  const int num_tiles = p.m_tiles * p.n_tiles;
  const int num_units = (MODE == MODE_PLAIN) ? num_tiles * p.splits : num_tiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumerThreads / 32) {
    // ===== TMA producer =====
    if (lane == 0) {
      prefetch_tmap(&tmap_a);
      prefetch_tmap(&tmap_b);
      int stage = 0;
      uint32_t phase = 0;
      int ready_chunk = -1;
      for (int u = cta; u < num_units; u += n_gemm_ctas) {
        const int t = (MODE == MODE_PLAIN) ? u % num_tiles : u;
        int kb0 = 0, kb1 = k_blocks;
        if (MODE == MODE_PLAIN && p.splits > 1) {
          kb0 = (u / num_tiles) * p.kb_per_split;
          kb1 = kb0 + p.kb_per_split < k_blocks ? kb0 + p.kb_per_split : k_blocks;
        }
        int m_blk, n_blk, chunk;
        tile_coords<MODE>(t, p, fa, m_blk, n_blk, chunk);
        const CUtensorMap* bmap = &tmap_b;
        int b_row = n_blk * BN;
        if (MODE == MODE_AG) {
          const int c_lo = (n_blk * BN) / fa.ag_rows, c_hi = (n_blk * BN + BN - 1) / fa.ag_rows;
          if (c_lo == fa.f.me && c_hi == fa.f.me) {
            bmap = &cm.m[0];  // entirely inside my own shard: no transfer needed
            b_row = n_blk * BN - fa.f.me * fa.ag_rows;
          } else if (n_blk != ready_chunk) {
            for (int c = c_lo; c <= c_hi; ++c)
              spin_wait_gpu(fa.f.local + (fa.epoch ? F_AGCHUNK : F_CHUNK) + c, q);
            fence_proxy_async_all();
            ready_chunk = n_blk;
          }
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem_a + stage * kSmemABytes;
          uint8_t* sb = smem_b + stage * Cfg::kSmemBBytes;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (A_KMAJOR) {
            tma_load_2d(&tmap_a, &full_bar[stage], sa, kb * BK, m_blk * BM);
          } else {
            // MN-major: one 64(m) x 64(k) swizzle atom column per box
#pragma unroll
            for (int h = 0; h < BM / 64; ++h)
              tma_load_2d(&tmap_a, &full_bar[stage], sa + h * (64 * BK * 2), m_blk * BM + h * 64,
                          kb * BK);
          }
          if (B_KMAJOR) {
            tma_load_2d(bmap, &full_bar[stage], sb, kb * BK, b_row);
          } else {
#pragma unroll
            for (int h = 0; h < BN / 64; ++h)
              tma_load_2d(bmap, &full_bar[stage], sb + h * (64 * BK * 2), b_row + h * 64, kb * BK);
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===== consumer warpgroups: wgmma main loop, then registers -> bf16 -> swizzled smem -> TMA store
    const int wg = warp >> 2;
    const int tid = threadIdx.x & 127;
    const int frag_row = 16 * (tid >> 5) + ((tid & 31) >> 2);  // + 8 for the odd register pairs
    const int frag_col = 2 * (tid & 3);
    const int row0 = wg * 64 + frag_row;                       // tile row of h = 0
    const bool issuer = (threadIdx.x == 0);
    if (issuer) prefetch_tmap(&tmap_c);
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    int ebuf = 0;
    for (int u = cta; u < num_units; u += n_gemm_ctas) {
      const int t = (MODE == MODE_PLAIN) ? u % num_tiles : u;
      int kb0 = 0, kb1 = k_blocks;
      if (MODE == MODE_PLAIN && p.splits > 1) {
        kb0 = (u / num_tiles) * p.kb_per_split;
        kb1 = kb0 + p.kb_per_split < k_blocks ? kb0 + p.kb_per_split : k_blocks;
      }
      int m_blk, n_blk, chunk;
      tile_coords<MODE>(t, p, fa, m_blk, n_blk, chunk);

      // main loop: one wgmma group in flight; a stage goes back to the producer once the group
      // that read it has retired
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence();
        mma_k_block<BN, A_KMAJOR, B_KMAJOR>(acc, smem_u32(smem_a + stage * kSmemABytes) + wg * (64 * BK * 2),
                                            smem_u32(smem_b + stage * Cfg::kSmemBBytes), kb == kb0);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);

      if (MODE == MODE_PLAIN && p.splits > 1) {
        // split-K: this unit's fp32 partial goes straight from registers to the workspace;
        // k_splitk_reduce adds the slices and the bias, and rounds
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t r = (int64_t)m_blk * BM + row0 + 8 * h;
          if (r >= p.M) continue;
          float* prow = p.partial + ((int64_t)(u / num_tiles) * p.M + r) * p.ldp;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = n_blk * BN + 8 * j + frag_col;
            if (col < p.ldp)  // ldp = N rounded up to 4, col even: whole float2 pairs only
              *reinterpret_cast<float2*>(prow + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          }
        }
        continue;
      }
      const CUtensorMap* cmap = &tmap_c;
      int c_row = m_blk * BM;
      if (MODE == MODE_RS) {
        cmap = &cm.m[chunk];  // receive slot [me] of the rank that owns these rows
        c_row = (m_blk - chunk * (p.m_tiles / fa.f.n)) * BM;
      }
      if (MODE == MODE_PLAIN && p.push_n > 0) {
        const int owner = m_blk / p.push_mtc;
        cmap = &cm.m[owner];
        c_row = (m_blk - owner * p.push_mtc) * BM;
      }
      const bool has_aux = (MODE == MODE_PLAIN && p.epi_op != EPI_NONE);
#pragma unroll
      for (int c0 = 0; c0 < BN; c0 += 64) {  // unrolled: acc must only ever be indexed statically
        float* v = acc + c0 / 2;  // this thread's 32 values of columns [c0, c0 + 64)
        if (p.bias != nullptr) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = n_blk * BN + c0 + 8 * j + frag_col;
            if (col < p.N) {  // N % 8 == 0 whenever a bias is passed
              const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.bias + col));
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                v[4 * j + 2 * h] += f.x;
                v[4 * j + 2 * h + 1] += f.y;
              }
            }
          }
        }
        if (has_aux) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int64_t r = (int64_t)m_blk * BM + row0 + 8 * h;
            const __nv_bfloat16* arow = p.aux + r * p.ld_aux;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int col = n_blk * BN + c0 + 8 * j + frag_col;
              float2 f = make_float2(0.f, 0.f);
              if (r < p.M && col < p.N)
                f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(arow + col));
              float x0 = v[4 * j + 2 * h], x1 = v[4 * j + 2 * h + 1];
              if (p.epi_op == EPI_ADD) {
                x0 += f.x;
                x1 += f.y;
              } else {
                // ATen multiplies the bf16-rounded GEMM result: reproduce that rounding
                x0 = __bfloat162float(__float2bfloat16_rn(x0)) * gelu_tanh_grad(f.x);
                x1 = __bfloat162float(__float2bfloat16_rn(x1)) * gelu_tanh_grad(f.y);
              }
              v[4 * j + 2 * h] = x0;
              v[4 * j + 2 * h + 1] = x1;
            }
          }
        }
        // the staging buffer we are about to overwrite must have been read by its TMA store
        if (issuer) tma_store_wait_read<Cfg::kEpiBufs - 1>();
        epi_bar_sync();
        uint8_t* buf = smem_epi + ebuf * Cfg::kEpiBufBytes;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          uint8_t* rowp = buf + row * 128 + frag_col * 2;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            __nv_bfloat162 o = __floats2bfloat162_rn(v[4 * j + 2 * h], v[4 * j + 2 * h + 1]);
            // 128-byte swizzle: 16-byte chunk j of row r lives at chunk (j ^ (r & 7))
            *reinterpret_cast<__nv_bfloat162*>(rowp + ((j ^ (row & 7)) << 4)) = o;
          }
        }
        fence_proxy_async();
        epi_bar_sync();
        if (issuer) {
          tma_store_2d(cmap, buf, n_blk * BN + c0, c_row);
          tma_store_commit();
        }
        ebuf ^= 1;
      }
      if (MODE == MODE_RS && issuer) {
        // this tile now sits (or is in flight to) its owner: count it, and when the last tile of
        // the chunk has landed tell the owner that source `me` is complete
        tma_store_wait_all();
        fence_proxy_async_all();
        __threadfence_system();
        const unsigned long long prev_cnt = atomicAdd(
            reinterpret_cast<unsigned long long*>(fa.f.local + F_TILECNT + chunk), 1ULL);
        if (prev_cnt == (unsigned long long)fa.tiles_per_chunk - 1) {
          fa.f.local[F_TILECNT + chunk] = 0;
          __threadfence_system();
          st_release_sys(fa.f.peer[chunk] + (fa.rs_defer ? F_PUSHED : F_CHUNK) + fa.f.me, q);
        }
      }
    }
    if (issuer) {
      if (MODE == MODE_PLAIN && p.push_n > 0 && p.push_sync == 0) {
        tma_store_wait_read<0>();
      } else {
        tma_store_wait_all();
        if (MODE == MODE_PLAIN && p.push_n > 0 && p.push_sync >= 2) {
          // the tiles went into peer memory: make them visible system-wide before this CTA retires
          // (the next edb_epoch_barrier on the stream then orders them before its signal)
          fence_proxy_async_all();
          __threadfence_system();
        }
      }
    }
  }

  if (MODE == MODE_RS) {
    __syncthreads();
    if (fa.rs_defer) {
      if (blockIdx.x == 0 && threadIdx.x == 0) fa.rs_state[0] = q;  // read by k_rs_finish (later kernel)
    } else {
      // ===== tail: reduce my rows from the n receive slots (all local), rank order =====
      if (threadIdx.x < fa.f.n)
        spin_wait_sys(fa.f.local + F_CHUNK + threadIdx.x, q, fa.f.timeout_ns, fa.f.local + F_ERR);
      __syncthreads();
      const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
      const uint64_t nthr = (uint64_t)gridDim.x * blockDim.x;
      if (fa.rs_out_dtype == EDB_F32) rs_tail_reduce<float>(fa, tid, nthr);
      else rs_tail_reduce<__nv_bfloat16>(fa, tid, nthr);
    }
    finish_op(fa.f, q, &s_last, gridDim.x);
  }
}

// ---- k_gemm2_bf16: the plain single-GPU GEMM ---------------------------------------------------------
//
// C = A.B (+ bias, + fused epilogue) for launches that carry nothing else: no split-K, no prefetch
// CTAs, no push, 128 x 256 tiles.  Same tile, same smem ring, same MMA order per output element and
// the same epilogue arithmetic as k_gemm_bf16<256, .., MODE_PLAIN>, so the bits are the same; what
// differs is how the CTA is organised:
//   * 384 threads: warpgroup 0 produces (one lane issues TMA) and shrinks to 40 registers per
//     thread, warpgroups 1 and 2 consume and grow to 232: the 128 accumulator registers plus the
//     epilogue's temporaries fit, where the 168 of a 288-thread CTA spill;
//   * each consumer warpgroup stores its own 64 rows: 64 x 64 staging buffers, a 128-thread named
//     barrier and an elected thread of its own.  The warpgroups never wait for each other after the
//     main loop, so one may be storing while the other still multiplies.
// (CTA pairs that multicast their shared B tile were measured on top of this and were slower on
// most shapes of the GPT-2 step: DESIGN.md §6.  L2 operand traffic is not what limits this kernel.)
constexpr int kGemm2Threads = 384;
constexpr int kGemm2EpiBufBytes = 64 * 64 * 2;  // one 64 x 64 bf16 store box (128B swizzle)

template <int R> __device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R> __device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
// the two consumer warpgroups' named barriers (ids 1 and 2)
__device__ __forceinline__ void wg_bar_sync(int wg) {
  if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}
// mbar_wait for a kernel whose roles change their register budget: with a trap inside a role ptxas
// allocates the whole kernel at the launch-time budget (the 232-register consumers then spill like
// 168-register ones).  So the watchdog only reports here, the role winds down, and the kernel traps
// in the code all roles share.
__device__ __forceinline__ bool mbar_wait_ok(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  if (mbar_try_wait(addr, parity)) return true;
  const uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(addr, parity)) {
    if ((++spins & 0xfff) == 0 && globaltimer_ns() - t0 > 4000000000ull) return false;
  }
  return true;
}

template <bool A_KMAJOR, bool B_KMAJOR>
__global__ void __launch_bounds__(kGemm2Threads, 1)
    k_gemm2_bf16(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_c, const GemmParams p) {
  constexpr int BN = 256;
  using Cfg = TileCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kSmemABytes;
  uint8_t* smem_epi = smem + kStages * Cfg::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_epi + Cfg::kEpiBufs * Cfg::kEpiBufBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int wgi = threadIdx.x >> 7;
  const int k_blocks = (p.K + BK - 1) / BK;
  // tile t = (t % m_tiles, t / m_tiles); CTA c takes tiles c, c + grid, ... as k_gemm_bf16 does
  const int mt = p.m_tiles;
  const int num_units = mt * p.n_tiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  bool ok = true;  // false: a barrier wait ran into the watchdog
  if (wgi == 0) {
    // ===== TMA producer =====
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      prefetch_tmap(&tmap_a);
      prefetch_tmap(&tmap_b);
      int stage = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; ok && u < num_units; u += gridDim.x) {
        const int m_blk = u % mt, n_blk = u / mt;
        for (int kb = 0; kb < k_blocks; ++kb) {
          if (!(ok = mbar_wait_ok(&empty_bar[stage], phase ^ 1))) break;
          uint8_t* sa = smem_a + stage * kSmemABytes;
          uint8_t* sb = smem_b + stage * Cfg::kSmemBBytes;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (A_KMAJOR) {
            tma_load_2d(&tmap_a, &full_bar[stage], sa, kb * BK, m_blk * BM);
          } else {
#pragma unroll
            for (int h = 0; h < BM / 64; ++h)
              tma_load_2d(&tmap_a, &full_bar[stage], sa + h * (64 * BK * 2), m_blk * BM + h * 64,
                          kb * BK);
          }
          if (B_KMAJOR) {
            tma_load_2d(&tmap_b, &full_bar[stage], sb, kb * BK, n_blk * BN);
          } else {
#pragma unroll
            for (int h = 0; h < BN / 64; ++h)
              tma_load_2d(&tmap_b, &full_bar[stage], sb + h * (64 * BK * 2), n_blk * BN + h * 64,
                          kb * BK);
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===== consumer warpgroups =====
    setmaxnreg_inc<232>();
    const int wg = wgi - 1;
    const int tid = threadIdx.x & 127;
    const int frag_row = 16 * (tid >> 5) + ((tid & 31) >> 2);  // + 8 for the odd register pairs
    const int frag_col = 2 * (tid & 3);
    const int row0 = wg * 64 + frag_row;  // tile row of h = 0
    const bool issuer = (tid == 0);       // owns this warpgroup's TMA-store bulk groups
    uint8_t* epi = smem_epi + wg * (2 * kGemm2EpiBufBytes);
    if (issuer) prefetch_tmap(&tmap_c);
    const int epi_op = p.epi_op;
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    int ebuf = 0;
    for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
      const int m_blk = u % mt, n_blk = u / mt;
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        if (!(ok = mbar_wait_ok(&full_bar[stage], phase))) break;
        wgmma_fence();
        mma_k_block<BN, A_KMAJOR, B_KMAJOR>(acc, smem_u32(smem_a + stage * kSmemABytes) + wg * (64 * BK * 2),
                                            smem_u32(smem_b + stage * Cfg::kSmemBBytes), kb == 0);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      if (!ok) break;
      if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);

      // epilogue: the arithmetic and the rounding points of k_gemm_bf16
#pragma unroll
      for (int c0 = 0; c0 < BN; c0 += 64) {  // unrolled: acc must only ever be indexed statically
        float* v = acc + c0 / 2;  // this thread's 32 values of columns [c0, c0 + 64)
        if (p.bias != nullptr) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = n_blk * BN + c0 + 8 * j + frag_col;
            if (col < p.N) {  // N % 8 == 0 whenever a bias is passed
              const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.bias + col));
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                v[4 * j + 2 * h] += f.x;
                v[4 * j + 2 * h + 1] += f.y;
              }
            }
          }
        }
        if (epi_op != EPI_NONE) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int64_t r = (int64_t)m_blk * BM + row0 + 8 * h;
            const __nv_bfloat16* arow = p.aux + r * p.ld_aux;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int col = n_blk * BN + c0 + 8 * j + frag_col;
              float2 f = make_float2(0.f, 0.f);
              if (r < p.M && col < p.N)
                f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(arow + col));
              float x0 = v[4 * j + 2 * h], x1 = v[4 * j + 2 * h + 1];
              if (epi_op == EPI_ADD) {
                x0 += f.x;
                x1 += f.y;
              } else {
                // ATen multiplies the bf16-rounded GEMM result: reproduce that rounding
                x0 = __bfloat162float(__float2bfloat16_rn(x0)) * gelu_tanh_grad(f.x);
                x1 = __bfloat162float(__float2bfloat16_rn(x1)) * gelu_tanh_grad(f.y);
              }
              v[4 * j + 2 * h] = x0;
              v[4 * j + 2 * h + 1] = x1;
            }
          }
        }
        // the staging buffer we are about to overwrite must have been read by its TMA store
        if (issuer) tma_store_wait_read<1>();
        wg_bar_sync(wg);
        uint8_t* buf = epi + ebuf * kGemm2EpiBufBytes;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = frag_row + 8 * h;
          uint8_t* rowp = buf + row * 128 + frag_col * 2;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            __nv_bfloat162 o = __floats2bfloat162_rn(v[4 * j + 2 * h], v[4 * j + 2 * h + 1]);
            // 128-byte swizzle: 16-byte chunk j of row r lives at chunk (j ^ (r & 7))
            *reinterpret_cast<__nv_bfloat162*>(rowp + ((j ^ (row & 7)) << 4)) = o;
          }
        }
        fence_proxy_async();
        wg_bar_sync(wg);
        if (issuer) {
          tma_store_2d(&tmap_c, buf, n_blk * BN + c0, m_blk * BM + wg * 64);
          tma_store_commit();
        }
        ebuf ^= 1;
      }
    }
    if (issuer) tma_store_wait_all();
  }
  if (!ok) asm volatile("trap;");  // a protocol bug becomes a launch error, not a hung GPU
}

// ---- deferred reduce-scatter: reduce the receive slots of many pushed GEMMs in one launch -----------
constexpr int kRsMaxItems = 160;
constexpr int kRsFinishThreads = 256;
constexpr int64_t kRsFinishChunkVecs = 4096;  // 64 KiB of bf16 per slot and work unit

struct RsFinishItem {
  const char* recv;     // n slots of chunk_bytes (local)
  void* dst;            // [chunk_bytes / 2] elements of out_dtype
  int64_t chunk_bytes;
  uint64_t* state;      // [0] op number of the push, [1] op number of this reduction
};
struct RsFinishDesc {
  FlagCtx f;
  int local_only;  // epoch mode: an edb_epoch_barrier earlier on the stream replaced every handshake
  int n_items;
  float scale;
  int out_dtype;
  int first_unit[kRsMaxItems + 1];
  RsFinishItem it[kRsMaxItems];
};

// NSRC > 0: group size known at compile time, so that exactly NSRC x U 16-byte loads are in flight
// per thread (8 for every instantiation: the slots are read once, nothing is reused, the kernel
// lives on memory-level parallelism); NSRC == 0: any group size, one vector at a time.
template <int NSRC>
__global__ void __launch_bounds__(kRsFinishThreads, 4)
    k_rs_finish(const __grid_constant__ RsFinishDesc d) {
  __shared__ uint64_t s_q;
  __shared__ unsigned long long s_need;
  __shared__ int s_last;
  if (threadIdx.x == 0) {
    s_q = ld_relaxed_gpu(d.f.local + F_SEQ) + 1;
    s_need = 0;
  }
  __syncthreads();
  if (!d.local_only) {
    // every source must have landed its tiles of the latest push among the items (flags are
    // monotonic and a source's pushes complete in stream order, so the latest covers the earlier)
    unsigned long long need = 0;
    for (int i = threadIdx.x; i < d.n_items; i += blockDim.x) {
      const unsigned long long e = ld_relaxed_gpu(d.it[i].state);
      need = e > need ? e : need;
    }
    if (need) atomicMax(&s_need, need);
    __syncthreads();
    if ((int)threadIdx.x < d.f.n)
      spin_wait_sys(d.f.local + F_PUSHED + threadIdx.x, s_need, d.f.timeout_ns, d.f.local + F_ERR);
    __syncthreads();
  }
  const uint64_t q = s_q;
  const int total_units = d.first_unit[d.n_items];
  const int n = NSRC > 0 ? NSRC : d.f.n;
  constexpr int MAXS = NSRC > 0 ? NSRC : kMaxGroup;
  constexpr int U = NSRC > 0 ? (8 / NSRC > 0 ? 8 / NSRC : 1) : 1;
  for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
    int lo = 0, hi = d.n_items;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (d.first_unit[mid] <= u) lo = mid;
      else hi = mid;
    }
    const char* recv = d.it[lo].recv;
    void* dst = d.it[lo].dst;
    const int64_t chunk_bytes = d.it[lo].chunk_bytes;
    const int64_t nvec = chunk_bytes / 16;
    const int64_t v0 = (int64_t)(u - d.first_unit[lo]) * kRsFinishChunkVecs;
    const int64_t v1 = v0 + kRsFinishChunkVecs < nvec ? v0 + kRsFinishChunkVecs : nvec;
    for (int64_t i0 = v0 + threadIdx.x; i0 < v1; i0 += U * kRsFinishThreads) {
      uint4 raw[U][MAXS];
#pragma unroll
      for (int uu = 0; uu < U; ++uu) {
        const int64_t i = i0 + uu * kRsFinishThreads;
        if (i < v1) {
#pragma unroll
          for (int sidx = 0; sidx < MAXS; ++sidx)
            if (sidx < n)
              raw[uu][sidx] = __ldcs(reinterpret_cast<const uint4*>(recv + (int64_t)sidx * chunk_bytes + i * 16));
        }
      }
#pragma unroll
      for (int uu = 0; uu < U; ++uu) {
        const int64_t i = i0 + uu * kRsFinishThreads;
        if (i >= v1) break;
        float acc[8];
#pragma unroll
        for (int sidx = 0; sidx < MAXS; ++sidx) {
          if (sidx < n) {
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[uu][sidx]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 v = __bfloat1622float2(h[e]);
              if (sidx == 0) {
                acc[2 * e] = v.x;
                acc[2 * e + 1] = v.y;
              } else {
                acc[2 * e] += v.x;
                acc[2 * e + 1] += v.y;
              }
            }
          }
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] *= d.scale;
        if (d.out_dtype == EDB_F32) rs_store<float>(static_cast<float*>(dst), i, acc);
        else rs_store<__nv_bfloat16>(static_cast<__nv_bfloat16*>(dst), i, acc);
      }
    }
  }
  if (d.local_only) return;
  // remember which op reduced these slots (the next pushes check the owners' DONE against it)
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < d.n_items; i += blockDim.x) d.it[i].state[1] = q;
  finish_op(d.f, q, &s_last, gridDim.x);
}

// push mode: row r of C belongs to member r / rows_per and goes to base[owner] + (r % rows_per) * ldc
struct PushDst {
  int n;
  int64_t rows_per, row_rot;
  __nv_bfloat16* base[kMaxGroup];
};

__global__ void __launch_bounds__(256)
    k_splitk_reduce(__nv_bfloat16* __restrict__ C, int64_t ldc, const float* __restrict__ partial,
                    int64_t ldp, int splits, int M, int N, const __nv_bfloat16* __restrict__ bias,
                    const __grid_constant__ PushDst pd) {
  const int64_t groups_per_row = ldp / 4;
  const int64_t total = (int64_t)M * groups_per_row;
  const int64_t slice = (int64_t)M * ldp;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / groups_per_row;
    const int c = (int)(i - r * groups_per_row) * 4;
    if (pd.n > 0) r = (r + pd.row_rot) % M;  // start at the next member's rows (no incast)
    const float* src = partial + r * ldp + c;
    float4 acc = *reinterpret_cast<const float4*>(src);
    for (int s = 1; s < splits; ++s) {
      const float4 v = *reinterpret_cast<const float4*>(src + s * slice);
      acc.x += v.x;
      acc.y += v.y;
      acc.z += v.z;
      acc.w += v.w;
    }
    float o[4] = {acc.x, acc.y, acc.z, acc.w};
    __nv_bfloat16* dst = C + r * ldc + c;
    if (pd.n > 0) {
      const int64_t owner = r / pd.rows_per;
      dst = pd.base[owner] + (r - owner * pd.rows_per) * ldc + c;
    }
    if (c + 3 < N) {
      // whole group inside the row: one 8-byte store (ldc % 8 == 0 and c % 4 == 0 => aligned)
      if (bias) {
#pragma unroll
        for (int e = 0; e < 4; ++e) o[e] += __bfloat162float(bias[c + e]);
      }
      __nv_bfloat162 h0 = __floats2bfloat162_rn(o[0], o[1]);
      __nv_bfloat162 h1 = __floats2bfloat162_rn(o[2], o[3]);
      uint2 v;
      v.x = *reinterpret_cast<uint32_t*>(&h0);
      v.y = *reinterpret_cast<uint32_t*>(&h1);
      *reinterpret_cast<uint2*>(dst) = v;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (c + e < N) {
          if (bias) o[e] += __bfloat162float(bias[c + e]);
          dst[e] = __float2bfloat16_rn(o[e]);
        }
      }
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------------

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// 2-D bf16 tensor map: `inner` contiguous elements, `outer` rows `ld` elements apart.
static int make_tmap(CUtensorMap* map, const void* base, int64_t inner, int64_t outer, int64_t ld,
                     int box_inner, int box_outer) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error(EDB_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult rc = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS)
    return set_error(EDB_E_CUDA, "cuTensorMapEncodeTiled failed (%d) inner=%lld outer=%lld ld=%lld",
                     (int)rc, (long long)inner, (long long)outer, (long long)ld);
  return EDB_OK;
}

template <int BN, bool AK, bool BK_, int MODE>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                       const GemmParams& p, const FusedArgs& fa, const CMaps& cm, int grid,
                       cudaStream_t st) {
  using Cfg = TileCfg<BN>;
  static bool configured = false;
  auto kern = k_gemm_bf16<BN, AK, BK_, MODE>;
  if (!configured) {
    EDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    configured = true;
  }
  kern<<<grid, kGemmThreads, Cfg::kSmemBytes, st>>>(ta, tb, tc, p, fa, cm);
  count_launch();
  return cuda_check(cudaGetLastError(), "k_gemm_bf16 launch");
}

template <int MODE>
static int dispatch_gemm(int bn, bool a_k, bool b_k, const CUtensorMap& ta, const CUtensorMap& tb,
                         const CUtensorMap& tc, const GemmParams& p, const FusedArgs& fa,
                         const CMaps& cm, int grid, cudaStream_t st) {
  const int key = (bn == 256 ? 4 : 0) | (a_k ? 2 : 0) | (b_k ? 1 : 0);
  switch (key) {
    case 7: return launch_gemm<256, true, true, MODE>(ta, tb, tc, p, fa, cm, grid, st);
    case 6: return launch_gemm<256, true, false, MODE>(ta, tb, tc, p, fa, cm, grid, st);
    case 5: return launch_gemm<256, false, true, MODE>(ta, tb, tc, p, fa, cm, grid, st);
    case 4: return launch_gemm<256, false, false, MODE>(ta, tb, tc, p, fa, cm, grid, st);
    case 3: return launch_gemm<128, true, true, MODE>(ta, tb, tc, p, fa, cm, grid, st);
    case 2: return launch_gemm<128, true, false, MODE>(ta, tb, tc, p, fa, cm, grid, st);
    case 1: return launch_gemm<128, false, true, MODE>(ta, tb, tc, p, fa, cm, grid, st);
    default: return launch_gemm<128, false, false, MODE>(ta, tb, tc, p, fa, cm, grid, st);
  }
}

template <bool AK, bool BK_>
static int launch_gemm2(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                        const GemmParams& p, int grid, cudaStream_t st) {
  using Cfg = TileCfg<256>;
  static bool configured = false;
  auto kern = k_gemm2_bf16<AK, BK_>;
  if (!configured) {
    EDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    configured = true;
  }
  kern<<<grid, kGemm2Threads, Cfg::kSmemBytes, st>>>(ta, tb, tc, p);
  count_launch();
  return cuda_check(cudaGetLastError(), "k_gemm2_bf16 launch");
}

static int pick_bn(int64_t N) {
  // 256-wide tiles halve the A traffic per MMA (see TileCfg); 128 only where N leaves nothing
  // for the second half of a 256-wide tile
  return N <= 128 ? 128 : 256;
}

static int check_operands(const void* A, const void* B, const void* C, const void* bias, int64_t M,
                          int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc,
                          const char* who) {
  if (M <= 0 || N <= 0 || K <= 0) return set_error(EDB_E_UNSUPPORTED, "%s: empty problem", who);
  if (M > 0x7fffffff || N > 0x7fffffff || K > 0x7fffffff)
    return set_error(EDB_E_UNSUPPORTED, "%s: dimension too large", who);
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)C) & 15)
    return set_error(EDB_E_UNSUPPORTED, "%s: base pointers must be 16-byte aligned", who);
  // TMA: global strides must be multiples of 16 bytes; extents (M, N, K) may be anything — boxes
  // that run past an extent are zero-filled on load and clipped on store.
  if ((lda | ldb | ldc) & 7)
    return set_error(EDB_E_UNSUPPORTED, "%s: lda/ldb/ldc must be multiples of 8", who);
  if (bias && ((N & 7) || ((uintptr_t)bias & 15)))
    return set_error(EDB_E_UNSUPPORTED, "%s: bias needs N %% 8 == 0 and 16-byte alignment", who);
  return EDB_OK;
}

// fp32 workspace of split-K GEMMs: one slab per (device, stream) pair, allocated on first use and
// never freed, so a CUDA graph that captured a slab's address may replay at any later time.  The
// first use may come while the stream is being captured: torch.cuda.graph captures on a stream of its
// own, not on the one its eager warm-up ran on.
constexpr size_t kSplitKBytes = (size_t)64 << 20;
struct SplitKSlab {
  int device;
  cudaStream_t stream;
  float* ptr;
};
static SplitKSlab g_splitk[16];
static int g_splitk_n = 0;

static float* splitk_workspace(cudaStream_t st) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  for (int i = 0; i < g_splitk_n; ++i)
    if (g_splitk[i].device == dev && g_splitk[i].stream == st) return g_splitk[i].ptr;
  if (g_splitk_n == 16) return nullptr;
  // cudaMalloc enqueues nothing on `st`, so it is safe during a capture; a capture begun in the
  // (default) global mode forbids it unless this thread switches to relaxed mode for the call
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  if (cudaThreadExchangeStreamCaptureMode(&mode) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  float* ptr = nullptr;
  const cudaError_t err = cudaMalloc(&ptr, kSplitKBytes);
  cudaThreadExchangeStreamCaptureMode(&mode);  // restore the caller's mode
  if (err != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  g_splitk[g_splitk_n++] = {dev, st, ptr};
  return ptr;
}

static int sm_count_now() {
  Runtime& r = rt();
  if (!r.inited) {
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess)
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    r.sm_count = sms;
  }
  return r.sm_count;
}

}  // namespace edb

using namespace edb;

extern "C" {

// push: NULL, or the receive slots of the group members (C rows are spread over them)
struct PushSpec {
  int n, me;
  int64_t rows_per;          // M / n, a multiple of BM
  char* slot[kMaxGroup];     // member p's receive slot for MY rows: [rows_per, N] bf16, ld = N
};

// pf: NULL, or the all-gather prefetch that rides on this GEMM
// epi: NULL, or the fused elementwise epilogue
struct EpiSpec {
  int op;
  const void* aux;
  int64_t ld_aux;
};

struct PfSpec {
  int gid, n_items;
  const uint64_t* src_offs;
  const uint64_t* dst_offs;
  const int64_t* bytes;
  const int64_t* dst_strides;
  const int64_t* src_strides;  // may be NULL (all 0)
};

static int fill_prefetch(FusedArgs* fa, const PfSpec* pf, int want_ctas) {
  Runtime& r = rt();
  if (!r.inited) return set_error(EDB_E_STATE, "runtime not initialised (call edb_init)");
  if (pf->gid < 0 || pf->gid >= r.ngroups) return set_error(EDB_E_INVALID, "bad group id %d", pf->gid);
  if (pf->n_items < 0 || pf->n_items > kMaxPfItems)
    return set_error(EDB_E_UNSUPPORTED, "prefetch: at most %d items per launch", kMaxPfItems);
  const Group& g = r.groups[pf->gid];
  fa->f.n = g.n;
  fa->f.me = g.me;
  fa->pf_n = g.n;
  fa->pf_items = pf->n_items;
  fa->pf_local = r.heap;
  for (int p = 0; p < g.n; ++p) fa->pf_heap[p] = r.peer_heap[g.ranks[p]];
  int64_t blocks = 0;
  for (int i = 0; i < pf->n_items; ++i) {
    const int64_t b = pf->bytes[i], st = pf->dst_strides[i];
    if (b <= 0 || (b & 15) || (pf->src_offs[i] & 15) || (pf->dst_offs[i] & 15) || (st & 15) || st < b)
      return set_error(EDB_E_INVALID, "prefetch item %d: ranges must be 16-byte aligned, stride >= bytes", i);
    if (pf->src_offs[i] < kUserOffset || pf->src_offs[i] + (uint64_t)b > r.heap_bytes ||
        pf->dst_offs[i] < kUserOffset ||
        pf->dst_offs[i] + (uint64_t)st * (g.n - 1) + (uint64_t)b > r.heap_bytes)
      return set_error(EDB_E_INVALID, "prefetch item %d: symmetric range out of bounds", i);
    const int64_t sst = pf->src_strides ? pf->src_strides[i] : 0;
    if (sst < 0 || (sst & 15) ||
        pf->src_offs[i] + (uint64_t)sst * (g.n - 1) + (uint64_t)b > r.heap_bytes)
      return set_error(EDB_E_INVALID, "prefetch item %d: bad source stride", i);
    fa->pf_src[i] = pf->src_offs[i];
    fa->pf_dst[i] = pf->dst_offs[i];
    fa->pf_bytes[i] = b;
    fa->pf_stride[i] = st;
    fa->pf_sstride[i] = sst;
    fa->pf_inplace[i] = (sst == st && pf->src_offs[i] == pf->dst_offs[i]) ? 1 : 0;
    blocks += (b + 16383) / 16384 * (fa->pf_inplace[i] ? g.n - 1 : g.n);
  }
  int ctas = want_ctas;
  if (blocks < ctas) ctas = (int)blocks;
  if (ctas < 1 && blocks > 0) ctas = 1;
  fa->pf_ctas = pf->n_items > 0 ? ctas : 0;
  return EDB_OK;
}

static int gemm_plain_impl(void* C, const void* A, const void* B, const void* bias, int64_t M,
                           int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int a_kmajor,
                           int b_kmajor, void* stream, const PushSpec* push,
                           const PfSpec* pf = nullptr, const EpiSpec* epi = nullptr) {
  int rc = check_operands(A, B, C, bias, M, N, K, lda, ldb, ldc, "edb_gemm_bf16");
  if (rc) return rc;
  const int sms = sm_count_now();
  int bn = pick_bn(N);
  const bool forced_bn = rt().gemm_force_bn == 128 || rt().gemm_force_bn == 256;
  if (forced_bn) bn = (int)rt().gemm_force_bn;
  CUtensorMap ta, tb, tc;
  if (a_kmajor) rc = make_tmap(&ta, A, K, M, lda, BK, BM);
  else rc = make_tmap(&ta, A, M, K, lda, 64, BK);
  if (rc) return rc;
  GemmParams p;
  p.C = static_cast<__nv_bfloat16*>(C);
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.ldc = ldc;
  p.M = (int)M;
  p.N = (int)N;
  p.K = (int)K;
  p.m_tiles = (int)((M + BM - 1) / BM);
  p.n_tiles = (int)((N + bn - 1) / bn);
  p.push_n = 0;
  p.push_mtc = 1;
  p.m_rot = 0;
  p.push_sync = (int)rt().push_sync;
  p.aux = nullptr;
  p.ld_aux = 0;
  p.epi_op = EPI_NONE;
  if (epi && epi->op != EPI_NONE) {
    if (epi->op != EPI_ADD && epi->op != EPI_GELU_BWD)
      return set_error(EDB_E_INVALID, "edb_gemm_epi_bf16: unknown epilogue op %d", epi->op);
    if ((N & 7) || ((uintptr_t)epi->aux & 15) || (epi->ld_aux & 7) || epi->ld_aux < N || !epi->aux)
      return set_error(EDB_E_UNSUPPORTED,
                       "edb_gemm_epi_bf16: aux needs N %% 8 == 0, 16-byte alignment, ld %% 8 == 0");
    p.aux = static_cast<const __nv_bfloat16*>(epi->aux);
    p.ld_aux = epi->ld_aux;
    p.epi_op = epi->op;
  }
  FusedArgs fa;
  memset(&fa, 0, sizeof(fa));
  CMaps cm;
  memset(&cm, 0, sizeof(cm));
  PushDst pd;
  memset(&pd, 0, sizeof(pd));
  int sms_gemm = sms;  // SMs left to the GEMM when prefetch CTAs ride along
  if (pf && pf->n_items > 0) {
    int want = (int)rt().comm_ctas;
    if (want < 2) want = 2;
    if (want > sms / 4) want = sms / 4;
    rc = fill_prefetch(&fa, pf, want);
    if (rc) return rc;
    sms_gemm = sms - fa.pf_ctas;
  }
  if (push) {
    p.push_n = push->n;
    p.push_mtc = (int)(push->rows_per / BM);
    // start with the rows of the next member, end with my own (a local store)
    const int first_m = ((push->me + 1) % push->n) * p.push_mtc;
    p.m_rot = first_m;
    pd.n = push->n;
    pd.rows_per = push->rows_per;
    pd.row_rot = (int64_t)first_m * BM;
    for (int q = 0; q < push->n; ++q) {
      rc = make_tmap(&cm.m[q], push->slot[q], N, push->rows_per, N, 64, BM);
      if (rc) return rc;
      pd.base[q] = reinterpret_cast<__nv_bfloat16*>(push->slot[q]);
    }
  }
  p.splits = 1;
  p.kb_per_split = 0;
  p.partial = nullptr;
  p.ldp = (N + 3) / 4 * 4;
  cudaStream_t st = (cudaStream_t)stream;
  // split-K: when the tiles occupy at most half of the SMs and K is long (weight gradients:
  // M, N = layer widths, K = tokens), slices of K go to the idle SMs.  Each slice keeps >= 8
  // k-blocks so that the pipeline fill and the fp32 partial traffic stay small against the MMAs.
  const int units = p.m_tiles * p.n_tiles;
  const int ctas = units;
  const int k_blocks = (int)((K + BK - 1) / BK);
  if (rt().gemm_splitk && 2 * ctas <= sms_gemm && k_blocks >= 16 && p.epi_op == EPI_NONE) {
    int splits = sms_gemm / ctas;
    if (splits > k_blocks / 8) splits = k_blocks / 8;
    if (splits > 8) splits = 8;
    while (splits > 1 && (size_t)splits * (size_t)M * (size_t)p.ldp * sizeof(float) > kSplitKBytes)
      --splits;
    if (splits > 1) {
      float* ws = splitk_workspace(st);
      if (ws != nullptr) {
        p.kb_per_split = (k_blocks + splits - 1) / splits;
        p.splits = (k_blocks + p.kb_per_split - 1) / p.kb_per_split;  // no empty slice
        p.partial = ws;
      }
    }
  }
  // a launch that is nothing but a 128 x 256-tile GEMM runs k_gemm2_bf16.  What that kernel gains
  // is in the epilogue, a couple of k-blocks' worth of clocks per tile: past 256 k-blocks there is
  // under 1 % to win, and the one such GEMM of the GPT-2 step (LM-head dgrad, K = 50257) measured
  // 14 % slower with it, so those keep k_gemm_bf16 like everything that is not plain.
  const bool use2 = gemm2_enabled() && !push && fa.pf_ctas == 0 && p.splits == 1 && bn == 256 &&
                    !forced_bn && k_blocks <= 256;
  if (b_kmajor) rc = make_tmap(&tb, B, K, N, ldb, BK, bn);
  else rc = make_tmap(&tb, B, N, K, ldb, 64, BK);
  if (rc) return rc;
  rc = make_tmap(&tc, C, N, push ? push->rows_per : M, ldc, 64, use2 ? 64 : BM);
  if (rc) return rc;
  const int tiles = units * p.splits;
  int grid = tiles < sms_gemm ? tiles : sms_gemm;
  if (use2) {
    if (a_kmajor) return b_kmajor ? launch_gemm2<true, true>(ta, tb, tc, p, grid, st)
                                  : launch_gemm2<true, false>(ta, tb, tc, p, grid, st);
    return b_kmajor ? launch_gemm2<false, true>(ta, tb, tc, p, grid, st)
                    : launch_gemm2<false, false>(ta, tb, tc, p, grid, st);
  }
  grid += fa.pf_ctas;
  rc = dispatch_gemm<MODE_PLAIN>(bn, a_kmajor != 0, b_kmajor != 0, ta, tb, tc, p, fa, cm, grid, st);
  if (rc || p.splits == 1) return rc;
  const int64_t groups = (int64_t)M * (p.ldp / 4);
  int rgrid = (int)((groups + 255) / 256);
  if (rgrid > 4 * sms) rgrid = 4 * sms;
  k_splitk_reduce<<<rgrid, 256, 0, st>>>(p.C, ldc, p.partial, p.ldp, p.splits, (int)M, (int)N, p.bias,
                                        pd);
  count_launch();
  return cuda_check(cudaGetLastError(), "k_splitk_reduce launch");
}

int edb_gemm_bf16(void* C, const void* A, const void* B, const void* bias, int64_t M, int64_t N,
                  int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int a_kmajor, int b_kmajor,
                  int accumulate_into_c, void* stream) {
  if (accumulate_into_c) return set_error(EDB_E_UNSUPPORTED, "edb_gemm_bf16: accumulate_into_c");
  return gemm_plain_impl(C, A, B, bias, M, N, K, lda, ldb, ldc, a_kmajor, b_kmajor, stream, nullptr);
}

int edb_gemm_pf_bf16(void* C, const void* A, const void* B, const void* bias, int64_t M, int64_t N,
                     int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int a_kmajor, int b_kmajor,
                     int gid, int n_items, const uint64_t* src_offs, const uint64_t* dst_offs,
                     const int64_t* bytes, const int64_t* dst_strides, const int64_t* src_strides,
                     void* stream) {
  PfSpec pf = {gid, n_items, src_offs, dst_offs, bytes, dst_strides, src_strides};
  return gemm_plain_impl(C, A, B, bias, M, N, K, lda, ldb, ldc, a_kmajor, b_kmajor, stream, nullptr,
                         n_items > 0 ? &pf : nullptr);
}

int edb_gemm_epi_bf16(void* C, const void* A, const void* B, const void* bias, const void* aux,
                      int64_t ld_aux, int epi_op, int64_t M, int64_t N, int64_t K, int64_t lda,
                      int64_t ldb, int64_t ldc, int a_kmajor, int b_kmajor, int gid, int n_items,
                      const uint64_t* src_offs, const uint64_t* dst_offs, const int64_t* bytes,
                      const int64_t* dst_strides, const int64_t* src_strides, void* stream) {
  PfSpec pf = {gid, n_items, src_offs, dst_offs, bytes, dst_strides, src_strides};
  EpiSpec epi = {epi_op, aux, ld_aux};
  return gemm_plain_impl(C, A, B, bias, M, N, K, lda, ldb, ldc, a_kmajor, b_kmajor, stream, nullptr,
                         n_items > 0 ? &pf : nullptr, &epi);
}

int edb_ag_prefetch(int gid, int n_items, const uint64_t* src_offs, const uint64_t* dst_offs,
                    const int64_t* bytes, const int64_t* dst_strides, const int64_t* src_strides,
                    void* stream) {
  if (n_items <= 0) return EDB_OK;
  Runtime& r = rt();
  static bool configured = false;
  const int smem = kPfSlots * 16384 + 1024 + 128;
  if (!configured) {
    EDB_CUDA(cudaFuncSetAttribute(k_ag_prefetch, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  for (int done = 0; done < n_items; done += kMaxPfItems) {
    const int k = n_items - done < kMaxPfItems ? n_items - done : kMaxPfItems;
    PfSpec pf = {gid, k, src_offs + done, dst_offs + done, bytes + done, dst_strides + done,
                 src_strides ? src_strides + done : nullptr};
    FusedArgs fa;
    memset(&fa, 0, sizeof(fa));
    // nothing else needs the SMs: one CTA per SM (1 thread each drives a 5-deep 16 KiB ring)
    int rc = fill_prefetch(&fa, &pf, r.sm_count);
    if (rc) return rc;
    if (fa.pf_ctas == 0) continue;
    k_ag_prefetch<<<fa.pf_ctas, 32, smem, (cudaStream_t)stream>>>(fa);
    count_launch();
    rc = cuda_check(cudaGetLastError(), "k_ag_prefetch launch");
    if (rc) return rc;
  }
  return EDB_OK;
}

int edb_gemm_push_bf16(int gid, uint64_t recv_off, const void* A, const void* B, int64_t M,
                       int64_t N, int64_t K, int64_t lda, int64_t ldb, int a_kmajor, int b_kmajor,
                       void* stream) {
  Runtime& r = rt();
  if (!r.inited) return set_error(EDB_E_STATE, "runtime not initialised (call edb_init)");
  if (gid < 0 || gid >= r.ngroups) return set_error(EDB_E_INVALID, "bad group id %d", gid);
  const Group& g = r.groups[gid];
  const int n = g.n, me = g.me;
  if (M % n || (M / n) % BM)
    return set_error(EDB_E_UNSUPPORTED, "edb_gemm_push_bf16: rows per rank must be a multiple of 128");
  if (N & 7) return set_error(EDB_E_UNSUPPORTED, "edb_gemm_push_bf16: N must be a multiple of 8");
  const int64_t rows = M / n;
  const size_t chunk_bytes = (size_t)rows * N * 2;
  if (recv_off < kUserOffset || recv_off + chunk_bytes * n > r.heap_bytes || (recv_off & 1023))
    return set_error(EDB_E_INVALID, "edb_gemm_push_bf16: bad symmetric offset");
  PushSpec ps;
  memset(&ps, 0, sizeof(ps));
  ps.n = n;
  ps.me = me;
  ps.rows_per = rows;
  for (int q = 0; q < n; ++q)
    ps.slot[q] = r.peer_heap[g.ranks[q]] + recv_off + (size_t)me * chunk_bytes;
  // C itself is never written in push mode; my own slot stands in for the checks / the unused map
  return gemm_plain_impl(ps.slot[me], A, B, nullptr, M, N, K, lda, ldb, N, a_kmajor, b_kmajor, stream,
                         &ps);
}

static int ag_gemm_impl(int gid, void* C, const void* A, const void* bias, uint64_t b_shard_off,
                        uint64_t b_full_off, int64_t M, int64_t N, int64_t K, int64_t lda,
                        int64_t ldc, void* stream, int epoch) {
  FusedArgs fa;
  memset(&fa, 0, sizeof(fa));
  fa.epoch = epoch;
  int rc = fill_flagctx(&fa.f, gid);
  if (rc) return rc;
  Runtime& r = rt();
  const Group& g = r.groups[gid];
  const int n = g.n, me = g.me;
  if (N % n) return set_error(EDB_E_UNSUPPORTED, "edb_ag_gemm_bf16: N %% group size != 0");
  const int64_t rows = N / n;
  int bn = 0;
  if (N % 256 == 0) bn = 256;
  else if (N % 128 == 0) bn = 128;
  else return set_error(EDB_E_UNSUPPORTED, "edb_ag_gemm_bf16: N=%lld not a multiple of 128",
                        (long long)N);
  if (rows % 8)
    return set_error(EDB_E_UNSUPPORTED, "edb_ag_gemm_bf16: shard rows %lld not a multiple of 8",
                     (long long)rows);
  if (K & 7) return set_error(EDB_E_UNSUPPORTED, "edb_ag_gemm_bf16: K must be a multiple of 8");
  const size_t shard_bytes = (size_t)rows * K * 2;
  if (b_shard_off < kUserOffset || b_shard_off + shard_bytes > r.heap_bytes || (b_shard_off & 15) ||
      b_full_off < kUserOffset || b_full_off + shard_bytes * n > r.heap_bytes || (b_full_off & 1023))
    return set_error(EDB_E_INVALID, "edb_ag_gemm_bf16: bad symmetric offsets");
  const char* shard = r.heap + b_shard_off;
  char* full = r.heap + b_full_off;
  rc = check_operands(A, full, C, bias, M, N, K, lda, K, ldc, "edb_ag_gemm_bf16");
  if (rc) return rc;
  CUtensorMap ta, tb, tc;
  rc = make_tmap(&ta, A, K, M, lda, BK, BM);
  if (rc) return rc;
  rc = make_tmap(&tb, full, K, N, K, BK, bn);
  if (rc) return rc;
  rc = make_tmap(&tc, C, N, M, ldc, 64, BM);
  if (rc) return rc;
  CMaps cm;
  memset(&cm, 0, sizeof(cm));
  rc = make_tmap(&cm.m[0], shard, K, rows, K, BK, bn);
  if (rc) return rc;
  GemmParams p;
  p.C = static_cast<__nv_bfloat16*>(C);
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.ldc = ldc;
  p.M = (int)M;
  p.N = (int)N;
  p.K = (int)K;
  p.m_tiles = (int)((M + BM - 1) / BM);
  p.n_tiles = (int)(N / bn);
  p.splits = 1;
  p.kb_per_split = 0;
  p.partial = nullptr;
  p.ldp = 0;
  p.push_n = 0;
  p.push_mtc = 1;
  p.m_rot = 0;
  p.push_sync = 0;
  p.aux = nullptr;
  p.ld_aux = 0;
  p.epi_op = EPI_NONE;
  const int sms = r.sm_count;
  int n_comm = (int)r.comm_ctas;
  if (n_comm < 1) n_comm = 1;
  if (n_comm > sms / 4) n_comm = sms / 4;
  if (n == 1) n_comm = 1;
  fa.n_comm = n_comm;
  for (int pidx = 0; pidx < n; ++pidx) fa.shard_src[pidx] = r.peer_heap[g.ranks[pidx]] + b_shard_off;
  fa.shard_src[me] = shard;
  fa.full_dst = full;
  fa.shard_bytes = (int64_t)shard_bytes;
  fa.ag_rows = (int)rows;
  fa.ag_first_tile = (int)(((int64_t)me * rows) / bn);
  const int tiles = p.m_tiles * p.n_tiles;
  int gemm_ctas = sms - n_comm;
  if (gemm_ctas > tiles) gemm_ctas = tiles;
  return dispatch_gemm<MODE_AG>(bn, true, true, ta, tb, tc, p, fa, cm, gemm_ctas + n_comm,
                                (cudaStream_t)stream);
}

int edb_ag_gemm_bf16(int gid, void* C, const void* A, const void* bias, uint64_t b_shard_off,
                     uint64_t b_full_off, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldc,
                     void* stream) {
  return ag_gemm_impl(gid, C, A, bias, b_shard_off, b_full_off, M, N, K, lda, ldc, stream, 0);
}

int edb_ag_gemm_epoch_bf16(int gid, void* C, const void* A, const void* bias, uint64_t b_shard_off,
                           uint64_t b_full_off, int64_t M, int64_t N, int64_t K, int64_t lda,
                           int64_t ldc, void* stream) {
  return ag_gemm_impl(gid, C, A, bias, b_shard_off, b_full_off, M, N, K, lda, ldc, stream, 1);
}

static int gemm_rs_impl(int gid, void* dst, uint64_t recv_off, uint64_t state_off, bool defer,
                        const void* A, const void* B, int64_t M, int64_t N, int64_t K, int64_t lda,
                        int64_t ldb, int a_kmajor, int b_kmajor, float post_scale, int out_dtype,
                        void* stream);

int edb_gemm_rs_bf16(int gid, void* dst, uint64_t recv_off, const void* A, const void* B,
                     int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb, int a_kmajor,
                     int b_kmajor, float post_scale, int out_dtype, void* stream) {
  return gemm_rs_impl(gid, dst, recv_off, 0, false, A, B, M, N, K, lda, ldb, a_kmajor, b_kmajor,
                      post_scale, out_dtype, stream);
}

int edb_gemm_rs_push_bf16(int gid, uint64_t recv_off, uint64_t state_off, const void* A,
                          const void* B, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                          int a_kmajor, int b_kmajor, void* stream) {
  Runtime& r = rt();
  if (!r.inited) return set_error(EDB_E_STATE, "runtime not initialised (call edb_init)");
  if (state_off < kUserOffset || state_off + 16 > r.heap_bytes || (state_off & 15))
    return set_error(EDB_E_INVALID, "edb_gemm_rs_push_bf16: bad state offset");
  return gemm_rs_impl(gid, nullptr, recv_off, state_off, true, A, B, M, N, K, lda, ldb, a_kmajor,
                      b_kmajor, 1.0f, EDB_BF16, stream);
}

static int rs_finish_impl(int gid, int n_items, void* const* dsts, const uint64_t* recv_offs,
                          const uint64_t* state_offs, const int64_t* chunk_bytes, float post_scale,
                          int out_dtype, void* stream, int local_only);

int edb_rs_finish(int gid, int n_items, void* const* dsts, const uint64_t* recv_offs,
                  const uint64_t* state_offs, const int64_t* chunk_bytes, float post_scale,
                  int out_dtype, void* stream) {
  return rs_finish_impl(gid, n_items, dsts, recv_offs, state_offs, chunk_bytes, post_scale,
                        out_dtype, stream, 0);
}

int edb_rs_finish_local(int gid, int n_items, void* const* dsts, const uint64_t* recv_offs,
                        const int64_t* chunk_bytes, float post_scale, int out_dtype, void* stream) {
  return rs_finish_impl(gid, n_items, dsts, recv_offs, nullptr, chunk_bytes, post_scale, out_dtype,
                        stream, 1);
}

static int rs_finish_impl(int gid, int n_items, void* const* dsts, const uint64_t* recv_offs,
                          const uint64_t* state_offs, const int64_t* chunk_bytes, float post_scale,
                          int out_dtype, void* stream, int local_only) {
  if (n_items <= 0) return EDB_OK;
  if (out_dtype != EDB_BF16 && out_dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "edb_rs_finish: out dtype must be bf16 or f32");
  Runtime& r = rt();
  cudaStream_t st = (cudaStream_t)stream;
  int done = 0;
  while (done < n_items) {
    RsFinishDesc d;
    int rc = fill_flagctx(&d.f, gid);
    if (rc) return rc;
    const int n = d.f.n;
    d.local_only = local_only;
    d.scale = post_scale;
    d.out_dtype = out_dtype;
    d.first_unit[0] = 0;
    int k = 0;
    int64_t units = 0;
    for (; done < n_items && k < kRsMaxItems; ++done, ++k) {
      const int64_t cb = chunk_bytes[done];
      if (cb <= 0 || (cb & 15) || ((uintptr_t)dsts[done] & 15))
        return set_error(EDB_E_INVALID, "edb_rs_finish: item %d: chunk bytes / dst alignment", done);
      if (recv_offs[done] < kUserOffset || recv_offs[done] + (uint64_t)cb * n > r.heap_bytes ||
          (recv_offs[done] & 15) ||
          (!local_only && (state_offs[done] < kUserOffset || state_offs[done] + 16 > r.heap_bytes ||
                           (state_offs[done] & 15))))
        return set_error(EDB_E_INVALID, "edb_rs_finish: item %d: bad symmetric offset", done);
      d.it[k].recv = r.heap + recv_offs[done];
      d.it[k].dst = dsts[done];
      d.it[k].chunk_bytes = cb;
      d.it[k].state = local_only ? nullptr : reinterpret_cast<uint64_t*>(r.heap + state_offs[done]);
      units += (cb / 16 + kRsFinishChunkVecs - 1) / kRsFinishChunkVecs;
      if (units > 0x7fffffffLL) return set_error(EDB_E_UNSUPPORTED, "edb_rs_finish: too much work");
      d.first_unit[k + 1] = (int)units;
    }
    d.n_items = k;
    int grid = (int)(units < 4LL * r.sm_count ? units : 4LL * r.sm_count);
    switch (n) {
      case 2: k_rs_finish<2><<<grid, kRsFinishThreads, 0, st>>>(d); break;
      case 4: k_rs_finish<4><<<grid, kRsFinishThreads, 0, st>>>(d); break;
      case 8: k_rs_finish<8><<<grid, kRsFinishThreads, 0, st>>>(d); break;
      default: k_rs_finish<0><<<grid, kRsFinishThreads, 0, st>>>(d); break;
    }
    count_launch();
    rc = cuda_check(cudaGetLastError(), "k_rs_finish launch");
    if (rc) return rc;
  }
  return EDB_OK;
}

static int gemm_rs_impl(int gid, void* dst, uint64_t recv_off, uint64_t state_off, bool defer,
                        const void* A, const void* B, int64_t M, int64_t N, int64_t K, int64_t lda,
                        int64_t ldb, int a_kmajor, int b_kmajor, float post_scale, int out_dtype,
                        void* stream) {
  FusedArgs fa;
  memset(&fa, 0, sizeof(fa));
  int rc = fill_flagctx(&fa.f, gid);
  if (rc) return rc;
  Runtime& r = rt();
  const Group& g = r.groups[gid];
  const int n = g.n, me = g.me;
  if (M % n || (M / n) % BM)
    return set_error(EDB_E_UNSUPPORTED, "edb_gemm_rs_bf16: rows per rank must be a multiple of 128");
  if (N & 7) return set_error(EDB_E_UNSUPPORTED, "edb_gemm_rs_bf16: N must be a multiple of 8");
  if (out_dtype != EDB_BF16 && out_dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "edb_gemm_rs_bf16: out dtype must be bf16 or f32");
  const int64_t rows = M / n;
  const size_t chunk_bytes = (size_t)rows * N * 2;
  if (recv_off < kUserOffset || recv_off + chunk_bytes * n > r.heap_bytes || (recv_off & 1023))
    return set_error(EDB_E_INVALID, "edb_gemm_rs_bf16: bad symmetric offset");
  char* recv = r.heap + recv_off;
  rc = check_operands(A, B, recv, nullptr, M, N, K, lda, ldb, N, "edb_gemm_rs_bf16");
  if (rc) return rc;
  const int sms = r.sm_count;
  const int bn = pick_bn(N);
  CUtensorMap ta, tb, tc;
  if (a_kmajor) rc = make_tmap(&ta, A, K, M, lda, BK, BM);
  else rc = make_tmap(&ta, A, M, K, lda, 64, BK);
  if (rc) return rc;
  if (b_kmajor) rc = make_tmap(&tb, B, K, N, ldb, BK, bn);
  else rc = make_tmap(&tb, B, N, K, ldb, 64, BK);
  if (rc) return rc;
  CMaps cm;
  memset(&cm, 0, sizeof(cm));
  for (int pidx = 0; pidx < n; ++pidx) {
    // rows owned by member pidx land in ITS receive buffer, slot [me]
    char* slot = r.peer_heap[g.ranks[pidx]] + recv_off + (size_t)me * chunk_bytes;
    rc = make_tmap(&cm.m[pidx], slot, N, rows, N, 64, BM);
    if (rc) return rc;
  }
  tc = cm.m[me];
  GemmParams p;
  p.C = reinterpret_cast<__nv_bfloat16*>(recv);
  p.bias = nullptr;
  p.ldc = N;
  p.M = (int)M;
  p.N = (int)N;
  p.K = (int)K;
  p.m_tiles = (int)(M / BM);
  p.n_tiles = (int)((N + bn - 1) / bn);
  p.splits = 1;
  p.kb_per_split = 0;
  p.partial = nullptr;
  p.ldp = 0;
  p.push_n = 0;
  p.push_mtc = 1;
  p.m_rot = 0;
  p.push_sync = 0;
  p.aux = nullptr;
  p.ld_aux = 0;
  p.epi_op = EPI_NONE;
  fa.recv_base = recv;
  fa.chunk_bytes = (int64_t)chunk_bytes;
  fa.rs_dst = dst;
  fa.rs_scale = post_scale;
  fa.rs_out_dtype = out_dtype;
  fa.tiles_per_chunk = (p.m_tiles / n) * p.n_tiles;
  fa.rs_defer = defer ? 1 : 0;
  fa.rs_state = defer ? reinterpret_cast<uint64_t*>(r.heap + state_off) : nullptr;
  // fused tail: always a full grid — CTAs without a tile still take part in the tail reduction,
  // which is latency-bound when only a few CTAs read the receive slots (small weight gradients);
  // push-only: one CTA per tile
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = defer ? (tiles < sms ? tiles : sms) : sms;
  return dispatch_gemm<MODE_RS>(bn, a_kmajor != 0, b_kmajor != 0, ta, tb, tc, p, fa, cm, grid,
                                (cudaStream_t)stream);
}

}  // extern "C"
