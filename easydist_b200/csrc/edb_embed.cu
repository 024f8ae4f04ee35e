// Token and position embeddings, forward and backward, for the sharded-op kernel dispatch of
// libedb.so.
//
// Forward: y[r] = W[idx[r]] (a gather, exact), optionally followed by the position table,
// y[b, t] = T(float(W[idx[b, t]]) + float(P[pos[t]])): GPT-2's `wte(idx) + wpe(pos)` in one pass,
// bit-identical to aten.embedding (+ aten.add, which rounds the fp32 sum once).  Ids outside the table
// read zeros.  One read of the indexed rows, one write of y.
//
// Backward: g[v] = T(sum of dy[r] over the rows r with idx[r] == v), the sum in fp32 and in
// increasing r, deterministic (no float atomics) and without host synchronisation:
//   1. memset of the (id, tile) run table;
//   2. k_embed_tile_sort: one CTA per tile of kTile rows sorts the keys (id << 32 | r) of its rows in
//      shared memory (bitonic; the keys are unique, so the order is fully determined) and writes the
//      sorted row numbers and, for every id present in the tile, the [start, end) of its run;
//   3. k_embed_bwd: one warp per (id, column chunk) walks the tiles in order and each run in order,
//      i.e. the rows of that id in increasing r, and adds their dy in fp32.
// Modes: dense writes all V rows (zeros where nothing was indexed, and for padding_idx), what
// aten.embedding_dense_backward returns; accumulate adds the rounded sum into `acc` in place,
// acc[v] = T(float(acc[v]) + float(T(sum))), for indexed rows only (every other row of acc is neither
// read nor written): the tied LM-head gradient `add(mm_lm_wgrad, embedding_dense_backward(...))`.
// Ids outside [0, V) are skipped; the padding row gets zeros (dense) or is left alone (accumulate).
// 16-byte vectors when C, the row strides and every pointer allow it, scalar accesses otherwise.
#include <cuda_bf16.h>

#include "edb_internal.cuh"
#include "edb_vec.cuh"

namespace edb {

constexpr int kEmbedTile = 2048;       // rows sorted by one CTA
constexpr int kEmbedSortThreads = 1024;
constexpr int kEmbedWarps = 8;         // ids per CTA of the backward sum

template <typename T, int EPV>
__device__ __forceinline__ void emb_ld(const T* p, float* f) {
  if constexpr (EPV == 1) f[0] = VecT<T>::ld(p);
  else VecT<T>::unpack(__ldg(reinterpret_cast<const uint4*>(p)), f);
}

template <typename T, int EPV>
__device__ __forceinline__ void emb_st(T* p, const float* f) {
  if constexpr (EPV == 1) VecT<T>::st(p, f[0]);
  else *reinterpret_cast<uint4*>(p) = VecT<T>::pack(f);
}

// y [rows, C] = W[idx] (+ P[pos[r % T]]); W, P and y contiguous rows of C elements
template <typename T, typename I, int EPV>
__global__ void __launch_bounds__(256)
    k_embed_fwd(T* __restrict__ y, const T* __restrict__ w, const I* __restrict__ idx,
                const T* __restrict__ p, const I* __restrict__ pos, int64_t rows, int64_t C,
                int64_t V, int64_t Vp, int64_t T_) {
  const int64_t nv = C / EPV, n = rows * nv;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / nv, c = (i - r * nv) * EPV;
    const int64_t v = (int64_t)idx[r];
    float f[EPV];
    if (v >= 0 && v < V) emb_ld<T, EPV>(w + v * C + c, f);
    else {
#pragma unroll
      for (int e = 0; e < EPV; ++e) f[e] = 0.0f;
    }
    if (p != nullptr) {
      const int64_t q = (int64_t)pos[r % T_];
      if (q >= 0 && q < Vp) {
        float g[EPV];
        emb_ld<T, EPV>(p + q * C + c, g);
#pragma unroll
        for (int e = 0; e < EPV; ++e) f[e] = __fadd_rn(f[e], g[e]);
      }
    }
    emb_st<T, EPV>(y + r * C + c, f);
  }
}

// one CTA per tile of kEmbedTile rows: sorted row numbers -> rs[tile * kEmbedTile + p], and for
// every id v present, runs[v * tiles + tile] = [start, end) of its rows in that sorted order
template <typename I>
__global__ void __launch_bounds__(kEmbedSortThreads)
    k_embed_tile_sort(int* __restrict__ rs, int2* __restrict__ runs, const I* __restrict__ idx,
                      int64_t rows, int64_t V, int tiles) {
  __shared__ uint64_t keys[kEmbedTile];
  const int tile = blockIdx.x;
  const int64_t r0 = (int64_t)tile * kEmbedTile;
  for (int i = threadIdx.x; i < kEmbedTile; i += blockDim.x) {
    const int64_t r = r0 + i;
    uint64_t k = ~0ull;  // past the end, or an id outside [0, V): sorts last, never summed
    if (r < rows) {
      const int64_t v = (int64_t)idx[r];
      if (v >= 0 && v < V) k = ((uint64_t)v << 32) | (uint64_t)r;
    }
    keys[i] = k;
  }
  __syncthreads();
  for (int k = 2; k <= kEmbedTile; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < kEmbedTile; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const uint64_t a = keys[i], b = keys[ixj];
          if ((a > b) == ((i & k) == 0)) {
            keys[i] = b;
            keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < kEmbedTile; i += blockDim.x) {
    const uint64_t key = keys[i];
    if (key == ~0ull) continue;
    const uint32_t v = (uint32_t)(key >> 32);
    rs[r0 + i] = (int)(uint32_t)key;
    int2* run = runs + (int64_t)v * tiles + tile;
    if (i == 0 || (uint32_t)(keys[i - 1] >> 32) != v) run->x = i;
    if (i == kEmbedTile - 1 || keys[i + 1] == ~0ull || (uint32_t)(keys[i + 1] >> 32) != v)
      run->y = i + 1;
  }
}

// one warp per (id v, chunk of 32 * EPV columns): the rows of v in increasing r, summed in fp32
template <typename T, int EPV>
__global__ void __launch_bounds__(kEmbedWarps * 32)
    k_embed_bwd(T* __restrict__ out, int64_t ld_out, const T* __restrict__ dy, int64_t ld_dy,
                const int* __restrict__ rs, const int2* __restrict__ runs, int tiles, int64_t V,
                int64_t C, int64_t pad, int accumulate) {
  const int lane = threadIdx.x & 31;
  const int64_t v = (int64_t)blockIdx.x * kEmbedWarps + (threadIdx.x >> 5);
  const int64_t c = ((int64_t)blockIdx.y * 32 + lane) * EPV;
  if (v >= V || c >= C) return;
  T* o = out + v * ld_out + c;
  float s[EPV];
#pragma unroll
  for (int e = 0; e < EPV; ++e) s[e] = 0.0f;
  if (v == pad) {
    if (!accumulate) emb_st<T, EPV>(o, s);
    return;
  }
  bool any = false;
  for (int t = 0; t < tiles; ++t) {
    const int2 run = runs[v * tiles + t];
    const int* rt = rs + (int64_t)t * kEmbedTile;
    for (int q = run.x; q < run.y; ++q) {
      float f[EPV];
      emb_ld<T, EPV>(dy + (int64_t)rt[q] * ld_dy + c, f);
#pragma unroll
      for (int e = 0; e < EPV; ++e) s[e] = __fadd_rn(s[e], f[e]);
      any = true;
    }
  }
  if (!accumulate) {
    emb_st<T, EPV>(o, s);
  } else if (any) {
    float a[EPV];
    emb_ld<T, EPV>(o, a);
#pragma unroll
    for (int e = 0; e < EPV; ++e) a[e] = __fadd_rn(a[e], VecT<T>::rnd(s[e]));
    emb_st<T, EPV>(o, a);
  }
}

static int64_t embed_tiles(int64_t rows) { return (rows + kEmbedTile - 1) / kEmbedTile; }

static size_t embed_runs_bytes(int64_t rows, int64_t V) {
  return ((size_t)(embed_tiles(rows) * V * sizeof(int2)) + 255) / 256 * 256;
}

template <typename T, int EPV>
static void embed_fwd_launch(void* y, const void* w, const void* idx, const void* p, const void* pos,
                             int64_t rows, int64_t C, int64_t V, int64_t Vp, int64_t T_, int idx64,
                             cudaStream_t s) {
  const int64_t n = rows * (C / EPV);
  const unsigned grid = (unsigned)(n / 256 + 1 < 65535 * 16 ? n / 256 + 1 : 65535 * 16);
  if (idx64)
    k_embed_fwd<T, int64_t, EPV><<<grid, 256, 0, s>>>((T*)y, (const T*)w, (const int64_t*)idx,
                                                      (const T*)p, (const int64_t*)pos, rows, C, V,
                                                      Vp, T_);
  else
    k_embed_fwd<T, int, EPV><<<grid, 256, 0, s>>>((T*)y, (const T*)w, (const int*)idx, (const T*)p,
                                                  (const int*)pos, rows, C, V, Vp, T_);
}

template <typename T, int EPV>
static void embed_bwd_launch(void* out, int64_t ld_out, const void* dy, int64_t ld_dy, const int* rs,
                             const int2* runs, int tiles, int64_t V, int64_t C, int64_t pad,
                             int accumulate, cudaStream_t s) {
  const dim3 grid((unsigned)((V + kEmbedWarps - 1) / kEmbedWarps),
                  (unsigned)((C + 32 * EPV - 1) / (32 * EPV)));
  k_embed_bwd<T, EPV><<<grid, kEmbedWarps * 32, 0, s>>>((T*)out, ld_out, (const T*)dy, ld_dy, rs,
                                                        runs, tiles, V, C, pad, accumulate);
}

}  // namespace edb

using namespace edb;

extern "C" {

int edb_embedding_fwd(void* y, const void* weight, const void* idx, const void* pos_weight,
                      const void* pos, int64_t rows, int64_t C, int64_t V, int64_t Vp, int64_t T,
                      int idx_dtype, int dtype, void* stream) {
  if (dtype != EDB_BF16 && dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "embedding_fwd: dtype %d", dtype);
  if (idx_dtype != EDB_I32 && idx_dtype != EDB_I64)
    return set_error(EDB_E_UNSUPPORTED, "embedding_fwd: index dtype %d", idx_dtype);
  if (rows < 0 || C < 1 || V < 0 || (pos_weight != nullptr && (pos == nullptr || T < 1 || Vp < 0)))
    return set_error(EDB_E_INVALID, "embedding_fwd: rows=%lld C=%lld V=%lld Vp=%lld T=%lld",
                     (long long)rows, (long long)C, (long long)V, (long long)Vp, (long long)T);
  if (pos_weight != nullptr && rows % T)
    return set_error(EDB_E_INVALID, "embedding_fwd: rows %lld not a multiple of T %lld",
                     (long long)rows, (long long)T);
  if (rows == 0) return EDB_OK;
  if (!y || !weight || !idx) return set_error(EDB_E_INVALID, "embedding_fwd: null pointer");
  const int es = dtype == EDB_BF16 ? 2 : 4, epv = 16 / es;
  const bool vec = C % epv == 0 &&
                   !(((uintptr_t)y | (uintptr_t)weight | (uintptr_t)pos_weight) & 15);
  const int idx64 = idx_dtype == EDB_I64;
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == EDB_BF16) {
    if (vec) embed_fwd_launch<__nv_bfloat16, 8>(y, weight, idx, pos_weight, pos, rows, C, V, Vp, T, idx64, s);
    else embed_fwd_launch<__nv_bfloat16, 1>(y, weight, idx, pos_weight, pos, rows, C, V, Vp, T, idx64, s);
  } else {
    if (vec) embed_fwd_launch<float, 4>(y, weight, idx, pos_weight, pos, rows, C, V, Vp, T, idx64, s);
    else embed_fwd_launch<float, 1>(y, weight, idx, pos_weight, pos, rows, C, V, Vp, T, idx64, s);
  }
  count_launch();
  return cuda_check(cudaGetLastError(), "k_embed_fwd launch");
}

int edb_embedding_bwd_workspace(int64_t rows, int64_t V, size_t* bytes_out) {
  if (rows < 0 || V < 0 || bytes_out == nullptr)
    return set_error(EDB_E_INVALID, "embedding_bwd_workspace: rows=%lld V=%lld", (long long)rows,
                     (long long)V);
  *bytes_out = embed_runs_bytes(rows, V) + (size_t)embed_tiles(rows) * kEmbedTile * sizeof(int);
  return EDB_OK;
}

int edb_embedding_bwd(void* out, int64_t ld_out, const void* dy, int64_t ld_dy, const void* idx,
                      void* workspace, int64_t rows, int64_t C, int64_t V, int64_t padding_idx,
                      int accumulate, int idx_dtype, int dtype, void* stream) {
  if (dtype != EDB_BF16 && dtype != EDB_F32)
    return set_error(EDB_E_UNSUPPORTED, "embedding_bwd: dtype %d", dtype);
  if (idx_dtype != EDB_I32 && idx_dtype != EDB_I64)
    return set_error(EDB_E_UNSUPPORTED, "embedding_bwd: index dtype %d", idx_dtype);
  if (rows < 0 || C < 1 || V < 0 || ld_out < C || (rows > 0 && ld_dy < C))
    return set_error(EDB_E_INVALID, "embedding_bwd: rows=%lld C=%lld V=%lld ld_out=%lld ld_dy=%lld",
                     (long long)rows, (long long)C, (long long)V, (long long)ld_out,
                     (long long)ld_dy);
  if (rows >= (1LL << 31) || V >= (1LL << 31) || (C + 31) / 32 > 65535 ||
      (V + kEmbedWarps - 1) / kEmbedWarps >= (1LL << 31))
    return set_error(EDB_E_UNSUPPORTED, "embedding_bwd: rows=%lld V=%lld C=%lld too large",
                     (long long)rows, (long long)V, (long long)C);
  if (V == 0 || (accumulate && rows == 0)) return EDB_OK;
  if (!out || (rows > 0 && (!dy || !idx || !workspace)))
    return set_error(EDB_E_INVALID, "embedding_bwd: null pointer");
  const int es = dtype == EDB_BF16 ? 2 : 4, epv = 16 / es;
  const bool vec = C % epv == 0 && ld_out % epv == 0 && ld_dy % epv == 0 &&
                   !(((uintptr_t)out | (uintptr_t)dy) & 15);
  const int tiles = (int)embed_tiles(rows);
  int2* runs = (int2*)workspace;
  int* rs = (int*)((char*)workspace + embed_runs_bytes(rows, V));
  cudaStream_t s = (cudaStream_t)stream;
  if (tiles > 0) {
    EDB_CUDA(cudaMemsetAsync(runs, 0, (size_t)tiles * V * sizeof(int2), s));
    if (idx_dtype == EDB_I64)
      k_embed_tile_sort<int64_t><<<tiles, kEmbedSortThreads, 0, s>>>(rs, runs, (const int64_t*)idx,
                                                                      rows, V, tiles);
    else
      k_embed_tile_sort<int><<<tiles, kEmbedSortThreads, 0, s>>>(rs, runs, (const int*)idx, rows, V,
                                                                  tiles);
    count_launch();
  }
  if (dtype == EDB_BF16) {
    if (vec) embed_bwd_launch<__nv_bfloat16, 8>(out, ld_out, dy, ld_dy, rs, runs, tiles, V, C, padding_idx, accumulate, s);
    else embed_bwd_launch<__nv_bfloat16, 1>(out, ld_out, dy, ld_dy, rs, runs, tiles, V, C, padding_idx, accumulate, s);
  } else {
    if (vec) embed_bwd_launch<float, 4>(out, ld_out, dy, ld_dy, rs, runs, tiles, V, C, padding_idx, accumulate, s);
    else embed_bwd_launch<float, 1>(out, ld_out, dy, ld_dy, rs, runs, tiles, V, C, padding_idx, accumulate, s);
  }
  count_launch();
  return cuda_check(cudaGetLastError(), "k_embed_bwd launch");
}

}  // extern "C"
