// Plane-native dense pipeline on Hopper tensor cores: fp32-accurate GEMMs whose operands AND results live in HBM as
// pre-split hi/lo planes (plane_fmt.cuh), so no conversion pass sits between the layers of a subnetwork.
//
// Two plane formats share one kernel template:
//   FMT_F16  (default)  hi = fp16(T), lo' = fp16((T - hi) 2^11); 2 B / value, k-block = 64 columns;
//                       wgmma m64n64k16 f16, C = sum a_hi b_hi + 2^-11 sum (a_hi b_lo' + a_lo' b_hi)
//   FMT_TF32 (fallback) hi = rna_tf32(T), lo = rna_tf32(T - hi); 4 B / value, k-block = 32 columns;
//                       mma.sync m16n8k8 tf32, C = sum a_hi b_hi + sum (a_hi b_lo + a_lo b_hi)
// Both carry 22 significant bits per value and drop only the lo*lo term (2^-22 relative).
//
// Planes of T[rows, cols] are k-block-major  plane[cols/BK][rows][BK]  (one 128 B row per (k-block, row)),
// zero padded in cols, followed by sign bits  bits[cols/32][rows]  (the ReLU mask of the backward pass costs
// 1/32..1/16 of a plane instead of a 4 B/element read).  One layout serves every GEMM of training because
// TMA can cut an operand tile out of the planes in either majorness:
//     K  = cols of T : box {BK, R rows, 1 kb}      -> K-major  [R rows][BK]          SWIZZLE_128B
//     K  = rows of T : box {BK, BK rows, R/BK kb}  -> MN-major [R/BK][BK k][BK mn]   SWIZZLE_128B
//   R = 128 for the A operand (tile rows), 64 for the B operand (tile columns).
//     fwd  Y = X W       A = Xp  K-major (K=in)    B = Wp  MN-major (N=out, K=in)
//     dX   = dZ W^T      A = dZp K-major (K=out)   B = Wp  K-major  (N=in,  K=out)
//     dW   = X^T dZ      A = Xp  MN-major (M=in)   B = dZp MN-major (N=out), K = batch
//   -> no transposed copies, and the epilogue of one GEMM writes the planes the
//   next one reads (bias+ReLU for fwd, ReLU mask + column sums for dX).
// wgmma takes fp16 operands in either majorness (the transpose bits of the instruction); its tf32 form takes K-major
// operands only, so the TF32 planes are multiplied with mma.sync from fragments read out of the same swizzled tiles.
//
// The tensor core's fp32 accumulation does not round to nearest, so hi*hi partial sums are kept in the MMA
// accumulator for 128 K only and then added into a separate register accumulator with RN; cross terms likewise.
//
// Kernel (pl_gemm_kernel): persistent, grouped, 512 threads = TMA producer warpgroup + 2 consumer warpgroups of 64
// rows of a 128 x 64 tile + an epilogue warpgroup.  The consumers write each finished tile's accumulators into one of
// two swizzled 32 KiB staging tiles and go on with the next tile's mainloop; the epilogue warpgroup reads the tile
// back row-per-lane and runs bias/ReLU/dropout, masks, column sums and the stores (fp16 plane tiles leave by TMA).
// The epilogue is the pace-setter of the thin-K waves, so its per-tile chain is kept short: the accumulators stay in
// registers, the global words a tile needs (ReLU mask, dropout step) are loaded one work item ahead, and each warp
// has a hi and a lo' store slab, so a slice never waits for a TMA store it has just issued.
// setmaxnreg gives the producer 40 registers and the rest to the consumers and the epilogue.
//
// Reference arithmetic replaced: tf.layers.dense and its gradients,
//   adanet/examples/simple_dnn.py:72-86,103-110.
#include <cuda.h>
#include <cudaTypedefs.h>

#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "dense_simt.cuh"
#include "planes.cuh"
#include "wgmma.cuh"

namespace adn {
namespace pl {

static constexpr int BM = 128, BN = 64;
static constexpr int STAGES = 3;
static constexpr int A_TILE = BM * 128;               // 16 KiB: 128 rows x one 128 B k-block row
static constexpr int B_TILE = BN * 128;               // 8 KiB
static constexpr int STAGE_BYTES = 2 * A_TILE + 2 * B_TILE;   // A_hi A_lo B_hi B_lo
static constexpr int CONSUMERS = 2;                   // consumer warpgroups, 64 tile rows each
static constexpr int CONSUMER_WARPS = 4 * CONSUMERS;
static constexpr int EPI_WARPS = 4;                   // the epilogue warpgroup: 32 tile rows per warp
static constexpr int NUM_THREADS = 128 * (1 + CONSUMERS) + 32 * EPI_WARPS;
// registers per thread after setmaxnreg: 128 (40 + EPI_REGS) + 256 CONSUMER_REGS <= 65536
static constexpr int PRODUCER_REGS = 40, EPI_REGS = 136, CONSUMER_REGS = 168;
static_assert(128 * (PRODUCER_REGS + EPI_REGS) + 128 * CONSUMERS * CONSUMER_REGS <= 65536, "register file");
// every warp starts with 65536 / NUM_THREADS = 128: the producer gives registers back, the others take them
static_assert(PRODUCER_REGS < 65536 / NUM_THREADS && EPI_REGS > 65536 / NUM_THREADS &&
              CONSUMER_REGS > 65536 / NUM_THREADS, "setmaxnreg.dec / .inc");
// finished tiles go from the consumers to the epilogue warpgroup through ACC_BUFS [BM][BN] fp32 staging tiles
static constexpr int ACC_BUFS = 2;
static constexpr int ACC_TILE_FLOATS = BM * BN;
static constexpr int ACC_BYTES = ACC_BUFS * ACC_TILE_FLOATS * 4;
// each epilogue warp has two 2 KB slabs (32x16 floats): the hi and the lo' plane slab of the TMA stores, so that a
// slice's two stores go out back to back; the first slab also serves the dense transpose
static constexpr int EPI_STAGE_FLOATS = 32 * 16;
static constexpr int EPI_BYTES = EPI_WARPS * 2 * EPI_STAGE_FLOATS * 4;
static constexpr int BAR_BYTES = 256;
static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + ACC_BYTES + EPI_BYTES + BAR_BYTES;   // (+ alignment)
static_assert(SMEM_BYTES <= 232448, "shared memory per block");
static constexpr int MAX_SPLITS = 64;

template <int FMT> struct Fmt;
template <> struct Fmt<FMT_TF32> {
  static constexpr int BK = 32;          // columns per k-block (128 B)
  static constexpr int CHUNK = 4;        // k-blocks per accumulation chunk (K = 128)
};
template <> struct Fmt<FMT_F16> {
  static constexpr int BK = 64;
  static constexpr int CHUNK = 2;        // K = 128
};

enum { EPI_BIAS_ACT = 0, EPI_MASK = 1, EPI_PARTIAL = 2 };

struct GemmParams {
  int M, N;
  int tiles_m, tiles_n, splits;
  int tiles;             // tiles_m * tiles_n
  float inv_tiles, inv_tiles_n;   // reciprocals for the division-free item decode (counts stay far below 2^21)
  int total_kb;          // k-blocks over the whole K
  int kb_per_split;
  int a_mn, b_mn;        // operand majorness (0 = K-major box, 1 = MN-major box)
  int out_planes;        // 1: result written as split planes (out / out_lo / out_bits), 0: dense fp32
  // output: dense row-major (ldc) / split-K partial [split][M][N], or planes
  void* out;             // dense base | hi plane base
  void* out_lo;          // lo plane base (out_planes)
  int ldc;
  int out_nb32;          // planes: 32-column blocks of the (padded) output tensor
  const float* bias;     // EPI_BIAS_ACT (nullable)
  int act;
  uint32_t* out_bits;    // planes + EPI_BIAS_ACT: sign bits of the output
  const uint32_t* mask_bits;  // EPI_MASK (nullable): sign bits of a [M, N] tensor; out = bit ? out : 0
  float* colsum_part;    // EPI_MASK (nullable): [ceil(M/32)][colsum_ld] per-32-row column sums of out
  int colsum_ld;
  float out_mul;         // EPI_MASK / EPI_PARTIAL: result multiplied by this (un-scaling of gradient planes, 1/(1-rate) of dropout)
  unsigned int* ovf;     // sticky overflow word (fp16 planes)
  // EPI_BIAS_ACT with planes out: tf.layers.dropout on the output (drop_thresh 0 = none)
  uint32_t drop_thresh;  // keep iff hash >= thresh (= rate * 2^32)
  uint32_t drop_key0;    // seed * 0x9E3779B1 + layer * 0x85EBCA77 + 0x27D4EB2F  (the step term is added on the device)
  float drop_scale;      // 1 / (1 - rate)
  uint32_t drop_idx0;    // element index of row 0 (row0 * N): a row slice of the minibatch draws the full batch's mask
  const int64_t* drop_step;
};

// ---------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Bounded spin: a broken pipeline traps (CUDA error) instead of hanging the GPU box.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  long long t0 = 0;
  for (uint32_t it = 0;; ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) return;
    if ((it & 1023u) == 1023u) {
      long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000LL) __trap();   // ~2 s at 2 GHz
    }
  }
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint32_t bar, uint32_t dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// shared -> global tile store (bulk async-group completion); coordinates past the tensor bounds are clipped
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// all but the most recently committed store group have finished reading shared memory
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void sts_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void sts_v2(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void lds_v4(uint32_t addr, float& a, float& b, float& c, float& d) {
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(a), "=f"(b), "=f"(c), "=f"(d) : "r"(addr) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// work item -> (tile_m, tile_n, split).  n fastest so concurrently resident CTAs share A tiles.
struct Item {
  int m0, n0, kb0, nkb, split;
};
// q = n / d for 0 <= n < 2^21 with inv = 1.0f / d: (n + 0.5) / d is never within 1/(2d) of an integer, far more than the
// fp32 error of the product, so the truncation is exact.  (An integer division is ~20 instructions; every one of the 18
// warps of a CTA decodes every work item, and on the thin-K layer waves that was a quarter of the stall samples.)
__device__ __forceinline__ int fast_div(int n, float inv) { return (int)(((float)n + 0.5f) * inv); }

__device__ __forceinline__ Item decode_item(const GemmParams& g, int item) {
  Item it;
  it.split = (g.splits == 1) ? 0 : fast_div(item, g.inv_tiles);
  const int t = item - it.split * g.tiles;
  const int tm = (g.tiles_n == 1) ? t : fast_div(t, g.inv_tiles_n);
  it.m0 = tm * BM;
  it.n0 = (t - tm * g.tiles_n) * BN;
  it.kb0 = it.split * g.kb_per_split;
  it.nkb = min(g.total_kb, it.kb0 + g.kb_per_split) - it.kb0;
  return it;
}

__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

__device__ __forceinline__ void st_global_v8(void* p, const uint32_t (&w)[8]) {   // 32 B as two 16 B stores
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = make_uint4(w[0], w[1], w[2], w[3]);
  q[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// split 32 values of one row into the two TF32 planes and write them with 32 B per store pair (TF32 planes have no
// TMA store path: the fp16 planes leave through store_slice_tma below)
__device__ __forceinline__ void store_row32_tf32(const GemmParams& g, const float* a, int my_row, int cbase) {
  constexpr int BK = Fmt<FMT_TF32>::BK;
  const size_t poff = ((size_t)(cbase / BK) * g.M + my_row) * BK + (cbase % BK);
  uint32_t hw[32], lw[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    float h, l;
    split_tf32(a[j], h, l);
    hw[j] = __float_as_uint(h);
    lw[j] = __float_as_uint(l);
  }
  float* hp = reinterpret_cast<float*>(g.out) + poff;
  float* lp = reinterpret_cast<float*>(g.out_lo) + poff;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    st_global_v8(hp + 8 * q, reinterpret_cast<const uint32_t(&)[8]>(hw[8 * q]));
    st_global_v8(lp + 8 * q, reinterpret_cast<const uint32_t(&)[8]>(lw[8 * q]));
  }
}

// The same slice of fp16 planes, through shared memory and TMA.  With direct stores from the row-owning lanes every
// lane of a store instruction would touch a different 128 B line, which the load/store unit serialises into 16 B
// wavefronts.  Here a lane writes its row's 64 B of one plane into the warp's 2 KB staging
// slab (16 B chunks XOR-swizzled the way CU_TENSOR_MAP_SWIZZLE_64B expects: chunk ^= (row >> 1) & 3, conflict-free)
// and one lane hands the [32 rows][32 columns] box to the TMA unit.  Rows past M are clipped by the tensor map.
// The hi and lo' planes have a slab each, and every slice commits its hi store and then its lo' store, so before a
// slab is written `wait_group.read 1` only waits for the store issued from it one slice earlier, not for the one
// just issued.
// 32 values -> their fp16 hi and lo' plane words, two values per word
__device__ __forceinline__ void split_f16x32(const float* a, uint32_t (&w)[16], uint32_t (&lw)[16]) {
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const __half2 h2 = __floats2half2_rn(a[2 * q], a[2 * q + 1]);
    const float2 hf = __half22float2(h2);
    const __half2 l2 = __floats2half2_rn((a[2 * q] - hf.x) * 2048.0f, (a[2 * q + 1] - hf.y) * 2048.0f);
    w[q] = *reinterpret_cast<const uint32_t*>(&h2);
    lw[q] = *reinterpret_cast<const uint32_t*>(&l2);
  }
}
__device__ __forceinline__ void store_slice_tma(const CUtensorMap* o_hi, const CUtensorMap* o_lo, uint32_t slab_hi,
                                                uint32_t slab_lo, const float* a, int lane, int mrow0, int cbase) {
  uint32_t w[16], lw[16];
  split_f16x32(a, w, lw);
  const uint32_t roff = (uint32_t)lane * 64u, sw = ((uint32_t)lane >> 1) & 3u;
  if (lane == 0) bulk_wait_read1();        // the hi store of the previous slice has read slab_hi
  __syncwarp();
#pragma unroll
  for (uint32_t j = 0; j < 4; ++j) sts_v4(slab_hi + roff + ((j ^ sw) << 4), w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
  fence_async_smem();
  __syncwarp();
  if (lane == 0) {
    tma_store_3d(o_hi, slab_hi, cbase & 63, mrow0, cbase >> 6);
    bulk_commit();
    bulk_wait_read1();                     // the lo' store of the previous slice has read slab_lo
  }
  __syncwarp();
#pragma unroll
  for (uint32_t j = 0; j < 4; ++j) sts_v4(slab_lo + roff + ((j ^ sw) << 4), lw[4 * j], lw[4 * j + 1], lw[4 * j + 2], lw[4 * j + 3]);
  fence_async_smem();
  __syncwarp();
  if (lane == 0) {
    tma_store_3d(o_lo, slab_lo, cbase & 63, mrow0, cbase >> 6);
    bulk_commit();
  }
}

// Forward epilogue with planes out, WITHOUT a register transpose: lane = row keeps its 32 accumulators (bias already
// added by the caller), applies ReLU / dropout, forms the sign-bit word, splits pairs of values with packed conversions
// and hands its 32 columns of each plane to the slab + TMA store path (fp16) or writes them with direct 16 B stores
// (TF32: 128 B per plane).  A caller with its own fp16 store path passes it as `store16` (the maps and slabs unused).
template <int FMT, class Store16 = void>
__device__ __forceinline__ void emit_slice_fwd_planes(const GemmParams& g, float* a, uint32_t drop_step, int lane, int mrow0,
                                                      int cbase, const CUtensorMap* o_hi, const CUtensorMap* o_lo,
                                                      uint32_t slab_hi, uint32_t slab_lo, const Store16* store16 = nullptr) {
  const int my_row = mrow0 + lane;
  const int kbo = cbase >> 5;
  if (kbo >= g.out_nb32) return;                         // warp-uniform
  const uint32_t cmask = (cbase + 32 <= g.N) ? 0xffffffffu : ((cbase < g.N) ? ((1u << (g.N - cbase)) - 1u) : 0u);
  if (g.act == ADN_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) a[j] = fmaxf(a[j], 0.f);
  }
  if (g.drop_thresh != 0u) {
    // tf.layers.dropout in TRAIN mode (simple_dnn.py:80-81): x * 1/(1-rate) * keep; the mask is the counter-based hash
    // the oracle restates (oracle/adanet_oracle.py dropout_keep_mask): element index = (row0 + row) * out + col
    const uint32_t key = g.drop_key0 + drop_step * 0xC2B2AE3Du;
    const uint32_t base = g.drop_idx0 + (uint32_t)my_row * (uint32_t)g.N + (uint32_t)cbase;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      uint32_t x = (base + (uint32_t)j) ^ key;
      x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
      a[j] = (x >= g.drop_thresh) ? a[j] * g.drop_scale : 0.f;
    }
  }
  if (cmask != 0xffffffffu) {       // K padding of the next GEMM must be exact zeros
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (!((cmask >> j) & 1u)) a[j] = 0.f;
  }
  if constexpr (!std::is_void<Store16>::value) (*store16)(a);
  else if (FMT == FMT_F16) store_slice_tma(o_hi, o_lo, slab_hi, slab_lo, a, lane, mrow0, cbase);
  else if (my_row < g.M) store_row32_tf32(g, a, my_row, cbase);
  uint32_t bits = 0u;
#pragma unroll
  for (int j = 0; j < 32; ++j) bits |= (a[j] > 0.f) ? (1u << j) : 0u;
  if (my_row < g.M) g.out_bits[(size_t)kbo * g.M + my_row] = bits;
}

// One round of the column-sum butterfly below, at distance W.  W is a template argument so that every index into `a`
// is a constant: with the distance as a loop variable the inner loop stayed rolled, and `a` went to local memory.
template <int W>
__device__ __forceinline__ void colsum_round(float* a, int lane) {
  const bool upper = (lane & W) != 0;
#pragma unroll
  for (int j = 0; j < W; ++j) {
    const float x = a[j], y = a[j + W];
    const float mine = upper ? y : x;
    const float send = upper ? x : y;
    a[j] = mine + __shfl_xor_sync(0xffffffffu, send, W);
  }
}

// dX epilogue with planes out, without a register transpose: sign-bit ReLU mask, plane stores as in the forward
// epilogue (slab + TMA for fp16 or the caller's `store16`, direct stores from the row-owning lane for TF32), and the per-32-row column sums
// (the bias gradient of the layer below) by a butterfly over the warp: at distance w a lane keeps the half of its
// columns selected by bit w of its lane id and receives the partner's partial sums for them, so after five rounds
// lane l holds the sum of column l over the 32 rows (31 shuffles and adds per lane, fixed order).
template <int FMT, class Store16 = void>
__device__ __forceinline__ void emit_slice_mask_planes(const GemmParams& g, float* a, uint32_t mwq, int lane, int mrow0, int cbase,
                                                       const CUtensorMap* o_hi, const CUtensorMap* o_lo, uint32_t slab_hi,
                                                       uint32_t slab_lo, const Store16* store16 = nullptr) {
  const int my_row = mrow0 + lane;
  const int kbo = cbase >> 5;
  if (kbo >= g.out_nb32) return;                         // warp-uniform
  const uint32_t cmask = (cbase + 32 <= g.N) ? 0xffffffffu : ((cbase < g.N) ? ((1u << (g.N - cbase)) - 1u) : 0u);
  const uint32_t keep = (my_row < g.M) ? (mwq & cmask) : 0u;     // rows past M contribute nothing to the column sums
  if (g.out_mul != 1.0f) {
#pragma unroll
    for (int j = 0; j < 32; ++j) a[j] *= g.out_mul;
  }
  if (keep != 0xffffffffu) {
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (!((keep >> j) & 1u)) a[j] = 0.f;
  }
  if constexpr (!std::is_void<Store16>::value) (*store16)(a);
  else if (FMT == FMT_F16) store_slice_tma(o_hi, o_lo, slab_hi, slab_lo, a, lane, mrow0, cbase);
  else if (my_row < g.M) store_row32_tf32(g, a, my_row, cbase);
  if (g.colsum_part) {
    colsum_round<16>(a, lane);
    colsum_round<8>(a, lane);
    colsum_round<4>(a, lane);
    colsum_round<2>(a, lane);
    colsum_round<1>(a, lane);
    const int col = cbase + lane;
    if (col < g.colsum_ld) g.colsum_part[(size_t)(mrow0 >> 5) * g.colsum_ld + col] = a[0];
  }
}

// One 32-row x 32-column slice of a tile: lane = row holds its 32 accumulators a[0..31] (columns cbase..cbase+31,
// the bias already in them).  Plane outputs go to the two functions above.  Everything else is a dense fp32 output
// (the logits y, the conv stem's dense dX, the dW split-K partials): ReLU, or the scale and the sign-bit ReLU mask,
// are applied in the register layout, then the slice is transposed through `stage` (16 B chunks XOR-swizzled by row:
// conflict-free both ways) and written with lane = 4-column group of 8 rows, so every global access covers whole
// 32 B sectors.
template <int FMT, int EPI>
__device__ __forceinline__ void emit_slice(const GemmParams& g, const bool out_planes, float* a, uint32_t mwq, float* stage,
                                           int lane, int mrow0, int cbase, int rows_ok, float* dense, bool dense_vec,
                                           const CUtensorMap* o_hi, const CUtensorMap* o_lo, uint32_t drop_step) {
  // `stage` is the warp's hi slab; its lo' slab follows it
  if (EPI == EPI_BIAS_ACT && out_planes) {
    emit_slice_fwd_planes<FMT>(g, a, drop_step, lane, mrow0, cbase, o_hi, o_lo, smem_u32(stage),
                               smem_u32(stage + EPI_STAGE_FLOATS));
    return;
  }
  if (EPI == EPI_MASK && out_planes) {
    emit_slice_mask_planes<FMT>(g, a, mwq, lane, mrow0, cbase, o_hi, o_lo, smem_u32(stage), smem_u32(stage + EPI_STAGE_FLOATS));
    return;
  }
  constexpr int SW = 16;                   // staged columns per pass (2 KB per warp, two passes)
  constexpr int CH = SW / 4;               // 16 B chunks per staged row
  constexpr int RPI = 32 / CH;             // rows covered by one transposed instruction (8)
  const int cc = lane % CH;                // 16 B chunk (4 columns) this lane owns after the transpose
  const int rsub = lane / CH;
  const bool live = cbase < g.N && rows_ok > 0;   // warp-uniform
  if (EPI == EPI_BIAS_ACT) {
    if (g.act == ADN_ACT_RELU) {
#pragma unroll
      for (int j = 0; j < 32; ++j) a[j] = fmaxf(a[j], 0.f);
    }
  } else {
    if (g.out_mul != 1.0f) {
#pragma unroll
      for (int j = 0; j < 32; ++j) a[j] *= g.out_mul;
    }
    if (EPI == EPI_MASK) {
      // valid columns of this slice as a bit mask (warp-uniform); all ones for interior tiles
      const uint32_t cmask = (cbase + 32 <= g.N) ? 0xffffffffu : ((cbase < g.N) ? ((1u << (g.N - cbase)) - 1u) : 0u);
      const uint32_t keep = mwq & cmask;
      if (keep != 0xffffffffu) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (!((keep >> j) & 1u)) a[j] = 0.f;
      }
    }
  }
  // chunk swizzle by row: both the row-wise float4 writes and the transposed float4 reads are bank-conflict free
#define ADN_SWZ(r) (((r) >> 1) & 3)
  float cs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 32 / SW; ++h) {
    {
      float4* srow = reinterpret_cast<float4*>(stage + lane * SW);
#pragma unroll
      for (int jj = 0; jj < CH; ++jj)
        srow[jj ^ ADN_SWZ(lane)] = make_float4(a[h * SW + 4 * jj], a[h * SW + 4 * jj + 1], a[h * SW + 4 * jj + 2],
                                               a[h * SW + 4 * jj + 3]);
    }
    __syncwarp();
    if (live) {
      const int c4 = h * SW + cc * 4;       // column offset inside the 32-column slice
      const int col = cbase + c4;
      cs[0] = cs[1] = cs[2] = cs[3] = 0.f;
#pragma unroll
      for (int i = 0; i < 32 / RPI; ++i) {
        const int r = rsub + RPI * i;
        const bool rv = (rows_ok == 32) || (r < rows_ok);
        float4 t = reinterpret_cast<const float4*>(stage + r * SW)[cc ^ ADN_SWZ(r)];
        float v[4] = {t.x, t.y, t.z, t.w};
        if (EPI == EPI_MASK) {
#pragma unroll
          for (int k = 0; k < 4; ++k) cs[k] += rv ? v[k] : 0.f;
        }
        if (rv) {
          float* op = dense + (size_t)(mrow0 + r) * g.ldc + col;
          if (dense_vec && col + 3 < g.N) {
            *reinterpret_cast<float4*>(op) = make_float4(v[0], v[1], v[2], v[3]);
          } else {
#pragma unroll
            for (int k = 0; k < 4; ++k)
              if (col + k < g.N) op[k] = v[k];
          }
        }
      }
      if (EPI == EPI_MASK && g.colsum_part) {
        // rows of this lane: rsub + RPI*i; fold the lanes that own the same columns in a fixed order
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          cs[k] += __shfl_xor_sync(0xffffffffu, cs[k], 4);
          cs[k] += __shfl_xor_sync(0xffffffffu, cs[k], 8);
          cs[k] += __shfl_xor_sync(0xffffffffu, cs[k], 16);
        }
        if (rsub == 0) {
          float* cp = g.colsum_part + (size_t)(mrow0 >> 5) * g.colsum_ld + col;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (col + k < g.colsum_ld) cp[k] = cs[k];
        }
      }
    }
    __syncwarp();
  }
#undef ADN_SWZ
}

// ---------------------------------------------------------------------------------
// GEMM kernel (grouped): one persistent launch runs the tiles of up to MAX_GROUP independent GEMMs of
// the same epilogue kind -- the same layer of every candidate subnetwork of an AdaNet iteration -- so the
// launch, prologue and pipeline fill/drain are paid once per layer wave instead of once per candidate,
// and the short-K tiles of narrow candidates hide behind the long-K tiles of wide ones.
// Work items are numbered problem after problem; CTA c takes items c, c + grid, ... (every CTA gets the
// same share of every problem).  A group of one is the plain single-GEMM call.
// ---------------------------------------------------------------------------------
static constexpr int MAX_GROUP = 8;

struct alignas(64) Problem {
  CUtensorMap a_hi, a_lo, b_hi, b_lo;
  CUtensorMap o_hi, o_lo;   // fp16 output planes as [32 rows][32 columns] store boxes
  GemmParams g;
  int item0;             // first work item of this problem
  int pad_[3];
};
struct alignas(64) Group {
  Problem p[MAX_GROUP];
  int n;                 // problems
  int total_items;
};

// Multi-source forward: y = act(x_0 w_0 + sum_s x_s w_s + b), the dense layer over a concatenation of its inputs.
// Every piece is its own plane tensor zero-padded in its own K tail, so the K loop runs over sum_p ceil(in_p / BK)
// k-blocks and the producer switches descriptors at piece boundaries; the consumers and the epilogue do not see the
// pieces.  A separate parameter block and instantiation leave the single-source parameter block (Group) as it is.
static constexpr int MAX_SRCS = ADN_FWD_MAX_SRCS;     // pieces besides (xp, wp)
struct alignas(64) MsProblem {
  CUtensorMap a_hi, a_lo, b_hi, b_lo;       // piece 0: the op's own xp / wp
  CUtensorMap o_hi, o_lo;
  CUtensorMap src[MAX_SRCS][4];             // pieces 1..n_src: a_hi, a_lo, b_hi, b_lo
  GemmParams g;
  int item0;
  int n_src;
  int kb_end[MAX_SRCS + 1];                 // k-block at which piece p ends (cumulative); kb_end[n_src] = g.total_kb
};
struct alignas(64) MsGroup {
  MsProblem p[MAX_GROUP];
  int n;
  int total_items;
};
static_assert(sizeof(MsGroup) <= 32764, "kernel parameter space");

// advance `cur` to the problem that owns `item` (items are visited in increasing order).  `next0` caches the first item
// of the following problem in a register: the common case is one compare, not an indexed load from the parameter bank.
template <class G>
__device__ __forceinline__ int find_problem(const G& grp, int cur, int item, int& next0) {
  while (item >= next0) {
    ++cur;
    next0 = (cur + 1 < grp.n) ? grp.p[cur + 1].item0 : 0x7fffffff;
  }
  return cur;
}
template <class G>
__device__ __forceinline__ int first_next0(const G& grp) { return grp.n > 1 ? grp.p[1].item0 : 0x7fffffff; }

// One work item as the epilogue warpgroup sees it, with the global values its slices need: the ReLU-mask words of
// the lane's row for the two 32-column halves (EPI_MASK; all ones without a mask, 0 past M or the last 32-column
// block) and the dropout step (EPI_BIAS_ACT with dropout).
struct EpiItem {
  int p;                 // problem
  Item it;
  uint32_t mw0, mw1;
  uint32_t drop_step;
};
template <int EPI, class G>
__device__ __forceinline__ EpiItem epi_fetch(const G& grp, int& cur, int& next0, int item, int tile_row) {
  EpiItem e;
  cur = find_problem(grp, cur, item, next0);
  e.p = cur;
  const GemmParams& g = grp.p[cur].g;
  e.it = decode_item(g, item - grp.p[cur].item0);
  e.mw0 = e.mw1 = 0xffffffffu;
  if (EPI == EPI_MASK && g.mask_bits) {
    const int my_row = e.it.m0 + tile_row, kbo = e.it.n0 >> 5;
    const bool row_ok = my_row < g.M;
    e.mw0 = (row_ok && kbo < g.out_nb32) ? __ldg(g.mask_bits + (size_t)kbo * g.M + my_row) : 0u;
    e.mw1 = (row_ok && kbo + 1 < g.out_nb32) ? __ldg(g.mask_bits + (size_t)(kbo + 1) * g.M + my_row) : 0u;
  }
  e.drop_step = (EPI == EPI_BIAS_ACT && g.drop_thresh != 0u) ? (uint32_t)(*g.drop_step) : 0u;
  return e;
}

template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// float offset of (row, col) in a [BM][BN] accumulator staging tile: 16 B chunk ^= row % 8, so that both the
// consumers' fragment-layout float2 writes and the epilogue's row-per-lane float4 reads are bank-conflict free
__device__ __forceinline__ int acc_off(int row, int col) {
  return row * BN + ((((col >> 2) ^ row) & 7) | ((col >> 2) & 8)) * 4 + (col & 3);
}

// adds one 128-K chunk of the MMA accumulators into the register accumulator with fp32 RN
template <int FMT>
__device__ __forceinline__ void fold_chunk(float (&acc)[32], const float (&H)[32], const float (&S)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] += H[j];
  if (FMT == FMT_F16) {
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = fmaf(S[j], 1.0f / 2048.0f, acc[j]);   // lo' carries 2^11
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] += S[j];
  }
}

// One k-block of a consumer warpgroup on fp16 planes: 4 K steps of 16, each hi*hi into H and hi*lo' + lo'*hi into S
// (first: the chunk starts, the MMAs overwrite H and S).  The warpgroup's 64 A rows start 8 KiB into the A tiles in
// both majornesses; a K step advances 32 B inside a K-major 128 B row, 16 rows of 128 B in an MN-major tile.
// a_hi: the warpgroup's 64 rows of the A hi tile, with the lo' tile A_TILE after it; b_hi: the B hi tile, with the
// lo' tile B_TILE after it.
template <int A_MN, int B_MN>
__device__ __forceinline__ void f16_kblock_at(uint32_t a_hi, uint32_t b_hi, float (&H)[32], float (&S)[32], bool first) {
  const uint32_t a_lo = a_hi + A_TILE, b_lo = b_hi + B_TILE;
  constexpr uint32_t a_step = A_MN ? 2048u : 32u, b_step = B_MN ? 2048u : 32u;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t sd = (first && k == 0) ? 0u : 1u;
    const uint64_t dah = wg::desc_sw128(a_hi + k * a_step), dal = wg::desc_sw128(a_lo + k * a_step);
    const uint64_t dbh = wg::desc_sw128(b_hi + k * b_step), dbl = wg::desc_sw128(b_lo + k * b_step);
    wg::mma_f16_n64<A_MN, B_MN>(H, dah, dbh, sd);
    wg::mma_f16_n64<A_MN, B_MN>(S, dah, dbl, sd);
    wg::mma_f16_n64<A_MN, B_MN>(S, dal, dbh, 1u);
  }
}
// the same on one pipeline stage of pl_gemm_kernel (A_hi A_lo B_hi B_lo)
template <int A_MN, int B_MN>
__device__ __forceinline__ void f16_kblock(uint32_t st, int wgi, float (&H)[32], float (&S)[32], bool first) {
  f16_kblock_at<A_MN, B_MN>(st + (uint32_t)wgi * 8192u, st + 2 * A_TILE, H, S, first);
}

// byte offset of (row r, byte c) in a tile of 128 B rows written by TMA with SWIZZLE_128B (16 B chunk ^= row % 8)
__device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return (uint32_t)(r * 128 + ((((c >> 4) ^ r) & 7) << 4) + (c & 15));
}
// element (mn, k) of a TF32 operand tile: K-major [rows][32 k] or MN-major [rows/32][32 k][32 mn]
template <int MN>
__device__ __forceinline__ uint32_t tf32_off(int mn, int k) {
  return MN ? (uint32_t)((mn >> 5) * 4096) + sw128_off(k, 4 * (mn & 31)) : sw128_off(mn, 4 * k);
}
__device__ __forceinline__ void mma_tf32_16x8(float* d, const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// One k-block of one consumer warp on TF32 planes: rows [arow0, +16) of the tile x all BN columns, 4 K steps of 8,
// accumulated in the same fragment layout as the wgmma path.
template <int A_MN, int B_MN>
__device__ __forceinline__ void tf32_kblock(const uint8_t* st, int arow0, int lane, float (&H)[32], float (&S)[32]) {
  const uint8_t* ah = st;
  const uint8_t* al = st + A_TILE;
  const uint8_t* bh = st + 2 * A_TILE;
  const uint8_t* bl = bh + B_TILE;
  const int gid = lane >> 2, tq = lane & 3;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t fa_h[4], fa_l[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const uint32_t o = tf32_off<A_MN>(arow0 + gid + 8 * (e & 1), 8 * ks + tq + 4 * (e >> 1));
      fa_h[e] = *reinterpret_cast<const uint32_t*>(ah + o);
      fa_l[e] = *reinterpret_cast<const uint32_t*>(al + o);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t o0 = tf32_off<B_MN>(8 * j + gid, 8 * ks + tq), o1 = tf32_off<B_MN>(8 * j + gid, 8 * ks + tq + 4);
      const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(bh + o0), bh1 = *reinterpret_cast<const uint32_t*>(bh + o1);
      const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(bl + o0), bl1 = *reinterpret_cast<const uint32_t*>(bl + o1);
      mma_tf32_16x8(&H[4 * j], fa_h, bh0, bh1);
      mma_tf32_16x8(&S[4 * j], fa_h, bl0, bl1);
      mma_tf32_16x8(&S[4 * j], fa_l, bh0, bh1);
    }
  }
}
// The kernel body, shared by pl_gemm_kernel (Group) and pl_gemm_ms_kernel (MsGroup, forward only).
template <int FMT, int EPI, class G>
__device__ __forceinline__ void pl_gemm_body(const G& grp) {
  constexpr bool MS = std::is_same<G, MsGroup>::value;
  constexpr int BK = Fmt<FMT>::BK;
  constexpr int CHUNK = Fmt<FMT>::CHUNK;
  constexpr int A_MN = EPI == EPI_PARTIAL, B_MN = EPI != EPI_MASK;   // operand majorness of fwd / dX / dW
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles must sit on 1024 B boundaries
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* acc_stage = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);
  float* epi_stage = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + ACC_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + ACC_BYTES + EPI_BYTES);
  uint64_t* full_bar = bars;                       // [STAGES]  TMA -> consumers
  uint64_t* empty_bar = bars + STAGES;             // [STAGES]  consumers -> TMA, count CONSUMER_WARPS
  uint64_t* tile_full = bars + 2 * STAGES;         // [ACC_BUFS] consumers -> epilogue, count 128 CONSUMERS
  uint64_t* tile_empty = tile_full + ACC_BUFS;     // [ACC_BUFS] epilogue -> consumers, count 32 EPI_WARPS

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  const int n_items = grp.total_items;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), CONSUMER_WARPS);
    }
    for (int b = 0; b < ACC_BUFS; ++b) {
      mbar_init(smem_u32(&tile_full[b]), 128 * CONSUMERS);
      mbar_init(smem_u32(&tile_empty[b]), 32 * EPI_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == 1 && lane < grp.n) {       // every problem's descriptors: each CTA visits every problem
    tma_prefetch_desc(&grp.p[lane].a_hi);
    tma_prefetch_desc(&grp.p[lane].a_lo);
    tma_prefetch_desc(&grp.p[lane].b_hi);
    tma_prefetch_desc(&grp.p[lane].b_lo);
    if constexpr (MS) {
      for (int q = 0; q < grp.p[lane].n_src; ++q)
        for (int m = 0; m < 4; ++m) tma_prefetch_desc(&grp.p[lane].src[q][m]);
    }
  }
  __syncthreads();

  if (warp < 4) {
    // ================= TMA producer =================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 0 && lane == 0) {
      uint32_t s = 0, ph = 0;
      int cur = 0, next0 = first_next0(grp);
      const uint32_t smem0 = smem_u32(smem);
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        cur = find_problem(grp, cur, item, next0);
        const auto& pr = grp.p[cur];
        const GemmParams& g = pr.g;
        const Item it = decode_item(g, item - pr.item0);
        // multi-source: the piece q of k-block kc, its first k-block and its end.  Multi-source problems have one
        // split (kb0 = 0), k-blocks are visited in order and every piece has at least one, so q advances by at most
        // one per k-block and the parameter block is read only at piece boundaries.
        [[maybe_unused]] int q = 0, q_kb0 = 0, q_end = 0;
        if constexpr (MS) q_end = pr.kb_end[0];
        for (int kb = 0; kb < it.nkb; ++kb) {
          mbar_wait(smem_u32(&empty_bar[s]), ph ^ 1);
          const uint32_t fb = smem_u32(&full_bar[s]);
          mbar_expect_tx(fb, STAGE_BYTES);
          const uint32_t base = smem0 + s * STAGE_BYTES;
          int kc = it.kb0 + kb;
          const CUtensorMap *a_hi = &pr.a_hi, *a_lo = &pr.a_lo, *b_hi = &pr.b_hi, *b_lo = &pr.b_lo;
          if constexpr (MS) {       // kc inside its piece
            if (kc >= q_end) {
              ++q;
              q_kb0 = q_end;
              q_end = pr.kb_end[q];
            }
            if (q > 0) {
              kc -= q_kb0;
              a_hi = &pr.src[q - 1][0]; a_lo = &pr.src[q - 1][1];
              b_hi = &pr.src[q - 1][2]; b_lo = &pr.src[q - 1][3];
            }
          }
          // K-major box {BK, rows, 1 kb} at (0, row0, kc); MN-major box {BK, BK rows, rows/BK kb} at (0, kc*BK, mn0/BK)
          const int a1 = A_MN ? kc * BK : it.m0, a2 = A_MN ? (it.m0 / BK) : kc;
          const int b1 = B_MN ? kc * BK : it.n0, b2 = B_MN ? (it.n0 / BK) : kc;
          tma_load_3d(a_hi, fb, base, 0, a1, a2);
          tma_load_3d(a_lo, fb, base + A_TILE, 0, a1, a2);
          tma_load_3d(b_hi, fb, base + 2 * A_TILE, 0, b1, b2);
          tma_load_3d(b_lo, fb, base + 2 * A_TILE + B_TILE, 0, b1, b2);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  if (warp >= 4 * (1 + CONSUMERS)) {
    // ================= epilogue warpgroup =================
    // Walks the same items as the consumers.  Warp ew owns tile rows [32 ew, +32): it reads each of its two 32 x 32
    // slices back row per lane and emits it; the staging tile is released once both slices are in registers.
    setmaxnreg_inc<EPI_REGS>();
    const int ew = warp - 4 * (1 + CONSUMERS);
    float* stage = epi_stage + ew * 2 * EPI_STAGE_FLOATS;
    const int row = 32 * ew + lane;
    int cur = 0, next0 = first_next0(grp);
    // The global loads of a work item (mask words, dropout step) are issued one item ahead, before the wait for the
    // current tile, so that they are not on the epilogue's critical path.
    EpiItem nx{};
    if ((int)blockIdx.x < n_items) nx = epi_fetch<EPI>(grp, cur, next0, blockIdx.x, row);
    uint32_t tcount = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++tcount) {
      const EpiItem e = nx;
      if (item + (int)gridDim.x < n_items) nx = epi_fetch<EPI>(grp, cur, next0, item + gridDim.x, row);
      const GemmParams& g = grp.p[e.p].g;
      const Item& it = e.it;
      const uint32_t buf = tcount & 1u;
      mbar_wait(smem_u32(&tile_full[buf]), (tcount >> 1) & 1u);
      const float* tile = acc_stage + buf * ACC_TILE_FLOATS;
      const int mrow0 = it.m0 + 32 * ew;
      float* dense = reinterpret_cast<float*>(g.out);
      if (EPI == EPI_PARTIAL) dense += (size_t)it.split * g.M * g.N;
      const bool out_planes = g.out_planes != 0;
      const bool dense_vec = !out_planes && ((g.ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(dense) & 15) == 0);
      const int rows_ok = min(32, g.M - mrow0);          // warp-uniform; <= 0: nothing to write
      const uint32_t mw0 = e.mw0, mw1 = e.mw1;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const int cs = 32 * h;
        float acc[32];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 v = *reinterpret_cast<const float4*>(tile + acc_off(row, cs + 4 * q));
          acc[4 * q] = v.x; acc[4 * q + 1] = v.y; acc[4 * q + 2] = v.z; acc[4 * q + 3] = v.w;
        }
        if (h == 1) mbar_arrive(smem_u32(&tile_empty[buf]));
        // ---- tile output: this warp's 32 rows x 32 columns ----
        const int ncol0 = it.n0 + cs;
        const uint32_t mw = h ? mw1 : mw0;
        if (FMT == FMT_F16 && !out_planes) {     // the dense transpose reuses the hi slab: earlier TMA stores have read it
          if (lane == 0) bulk_wait_read0();
          __syncwarp();
        }
        emit_slice<FMT, EPI>(g, out_planes, acc, mw, stage, lane, mrow0, ncol0, rows_ok, dense, dense_vec, &grp.p[e.p].o_hi,
                             &grp.p[e.p].o_lo, e.drop_step);
      }
    }
    if (FMT == FMT_F16 && lane == 0) bulk_wait0();    // stores complete before the CTA (and its shared memory) goes away
    return;
  }

  // ================= consumer warpgroups 1..2 =================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wgi = warp / 4 - 1;                    // which 64 rows of the tile
  const int wq = warp & 3;                         // warp inside the warpgroup
  const int gid = lane >> 2, tq = lane & 3;        // accumulator fragment coordinates
  const uint32_t smem0 = smem_u32(smem);
  uint32_t s = 0, ph = 0;
  int cur = 0, next0 = first_next0(grp);
  uint32_t tcount = 0;
  float H[32], S[32];                              // MMA accumulators of one 128-K chunk
#pragma unroll
  for (int j = 0; j < 32; ++j) H[j] = S[j] = 0.f;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++tcount) {
    cur = find_problem(grp, cur, item, next0);
    const GemmParams& g = grp.p[cur].g;
    const Item it = decode_item(g, item - grp.p[cur].item0);
    float acc[32];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {       // the bias starts the accumulation
        const int col = it.n0 + 8 * j + 2 * tq + (e & 1);
        acc[4 * j + e] = (EPI == EPI_BIAS_ACT && g.bias && col < g.N) ? __ldg(g.bias + col) : 0.f;
      }
    for (int kb = 0; kb < it.nkb; ++kb) {
      const bool first = (kb % CHUNK) == 0;
      const bool last = (kb % CHUNK) == CHUNK - 1 || kb == it.nkb - 1;
      mbar_wait(smem_u32(&full_bar[s]), ph);
      if (FMT == FMT_F16) {
        wg::fence_regs(H);
        wg::fence_regs(S);
        wg::fence();
        f16_kblock<A_MN, B_MN>(smem0 + s * STAGE_BYTES, wgi, H, S, first);
        wg::commit();
        wg::wait<0>();
        wg::fence_regs(H);
        wg::fence_regs(S);
      } else {
        if (first) {
#pragma unroll
          for (int j = 0; j < 32; ++j) H[j] = S[j] = 0.f;
        }
        tf32_kblock<A_MN, B_MN>(smem + s * STAGE_BYTES, 64 * wgi + 16 * wq, lane, H, S);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&empty_bar[s]));     // this warp is done with the stage
      if (++s == STAGES) { s = 0; ph ^= 1; }
      if (last) fold_chunk<FMT>(acc, H, S);
    }
    // ---- hand the tile to the epilogue warpgroup: fragment layout into staging tile tcount % 2 ----
    const uint32_t buf = tcount & 1u;
    mbar_wait(smem_u32(&tile_empty[buf]), ((tcount >> 1) & 1u) ^ 1u);
    float* tile = acc_stage + buf * ACC_TILE_FLOATS;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int row = 64 * wgi + 16 * wq + gid, col = 8 * j + 2 * tq;
      *reinterpret_cast<float2*>(tile + acc_off(row, col)) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(tile + acc_off(row + 8, col)) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    mbar_arrive(smem_u32(&tile_full[buf]));
  }
}

template <int FMT, int EPI>
__global__ void __launch_bounds__(NUM_THREADS, 1)
pl_gemm_kernel(const __grid_constant__ Group grp) {
  pl_gemm_body<FMT, EPI>(grp);
}
template <int FMT>
__global__ void __launch_bounds__(NUM_THREADS, 1)
pl_gemm_ms_kernel(const __grid_constant__ MsGroup grp) {
  pl_gemm_body<FMT, EPI_BIAS_ACT>(grp);
}

// ---------------------------------------------------------------------------------
// Thin-K kernel (pl_thin_kernel): fp16 planes in and out, every problem one accumulation chunk (K <= 128) and one
// split -- the first-layer forward and the logits layer's dX of a training step.  Their tiles have one or two k-blocks
// of MMA work and a full epilogue each, so pl_gemm_kernel's single epilogue warpgroup sets their pace and its ring
// reloads the same A rows for every tile.  Here a work item is (problem, 128-row block, a run of up to THIN_RUN
// N tiles): the row block's A planes are loaded into shared memory once per item and the B tiles stream through a
// small ring.  Each tile is two units of 64 rows; unit u of the CTA goes to math warpgroup u % THIN_WGS, which runs
// its MMAs, folds them, transposes the result through its own staging area and emits it, one 32 x 32 slice per warp,
// with the functions pl_gemm_kernel's epilogue uses; each plane of the unit then leaves in one 64 x 64 TMA store.  The arithmetic is the same instruction sequence (bias start,
// f16_kblock, fold_chunk), the dropout hash is keyed by element index and the column sums are written per 32-row
// slice, so the results are bit-identical to pl_gemm_kernel's.  One producer warp issues the TMA loads.
// ---------------------------------------------------------------------------------
static constexpr int THIN_WGS = 3;                    // math warpgroups
static constexpr int THIN_THREADS = 128 * THIN_WGS + 32;
static constexpr int THIN_RUN = 4;                    // N tiles per work item at most (load balance)
static constexpr int THIN_STAGES = 2;
static constexpr int THIN_A_BYTES = Fmt<FMT_F16>::CHUNK * 2 * A_TILE;     // per k-block: A_hi, A_lo (128 rows)
static constexpr int THIN_B_STAGE = Fmt<FMT_F16>::CHUNK * 2 * B_TILE;     // per k-block: B_hi, B_lo (64 columns)
static constexpr int THIN_ACC_FLOATS = 64 * BN;                           // one warpgroup's 64 x 64 staging area
static constexpr int THIN_SLAB_WG = 2 * 64 * 128;                        // a warpgroup's hi and lo' [64][64] fp16 slabs
static constexpr int THIN_SLAB_BYTES = THIN_WGS * THIN_SLAB_WG;
static constexpr int THIN_SMEM_BYTES =
    1024 + THIN_A_BYTES + THIN_STAGES * THIN_B_STAGE + THIN_WGS * THIN_ACC_FLOATS * 4 + THIN_SLAB_BYTES + BAR_BYTES;
static_assert(THIN_SMEM_BYTES <= 232448, "shared memory per block");

// work items of one problem: 128-row blocks x runs of N tiles
__host__ __device__ __forceinline__ int thin_runs(int tiles_n) { return (tiles_n + THIN_RUN - 1) / THIN_RUN; }

template <int EPI>
__global__ void __launch_bounds__(THIN_THREADS, 1)
pl_thin_kernel(const __grid_constant__ Group grp) {
  constexpr int A_MN = 0, B_MN = EPI == EPI_BIAS_ACT;   // fwd: A K-major, B MN-major; dX: both K-major
  constexpr int BK = Fmt<FMT_F16>::BK;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t a_smem = smem_u32(smem);
  const uint32_t b_smem = a_smem + THIN_A_BYTES;
  float* acc_stage = reinterpret_cast<float*>(smem + THIN_A_BYTES + THIN_STAGES * THIN_B_STAGE);
  float* slabs = acc_stage + THIN_WGS * THIN_ACC_FLOATS;
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(slabs) + THIN_SLAB_BYTES);
  uint64_t* full_bar = bars;                       // [THIN_STAGES]  B tile loaded
  uint64_t* empty_bar = bars + THIN_STAGES;        // [THIN_STAGES]  both 64-row units of the tile done, count 8 warps
  uint64_t* a_full = bars + 2 * THIN_STAGES;       // the item's A rows loaded
  uint64_t* a_empty = a_full + 1;                  // every math warp done with them, count 4 THIN_WGS

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  const int n_items = grp.total_items;

  if (threadIdx.x == 0) {
    for (int s = 0; s < THIN_STAGES; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 8);
    }
    mbar_init(smem_u32(a_full), 1);
    mbar_init(smem_u32(a_empty), 4 * THIN_WGS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == 4 * THIN_WGS && lane < grp.n) {
    tma_prefetch_desc(&grp.p[lane].a_hi);
    tma_prefetch_desc(&grp.p[lane].a_lo);
    tma_prefetch_desc(&grp.p[lane].b_hi);
    tma_prefetch_desc(&grp.p[lane].b_lo);
  }
  __syncthreads();

  if (warp == 4 * THIN_WGS) {
    // ================= TMA producer =================
    if (lane == 0) {
      int cur = 0, next0 = first_next0(grp);
      uint32_t tile = 0, icount = 0;               // B tiles and items of this CTA so far
      for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++icount) {
        cur = find_problem(grp, cur, item, next0);
        const Problem& pr = grp.p[cur];
        const GemmParams& g = pr.g;
        const int runs = thin_runs(g.tiles_n), local = item - pr.item0;
        const int mb = local / runs, t0 = (local - mb * runs) * THIN_RUN;
        const int nt = min(THIN_RUN, g.tiles_n - t0);
        if (icount > 0) mbar_wait(smem_u32(a_empty), (icount - 1) & 1u);
        mbar_expect_tx(smem_u32(a_full), g.total_kb * 2 * A_TILE);
        for (int kb = 0; kb < g.total_kb; ++kb) {
          tma_load_3d(&pr.a_hi, smem_u32(a_full), a_smem + kb * 2 * A_TILE, 0, mb * BM, kb);
          tma_load_3d(&pr.a_lo, smem_u32(a_full), a_smem + kb * 2 * A_TILE + A_TILE, 0, mb * BM, kb);
        }
        for (int j = 0; j < nt; ++j, ++tile) {
          const uint32_t s = tile % THIN_STAGES, ph = (tile / THIN_STAGES) & 1u;
          mbar_wait(smem_u32(&empty_bar[s]), ph ^ 1u);
          const uint32_t fb = smem_u32(&full_bar[s]);
          mbar_expect_tx(fb, g.total_kb * 2 * B_TILE);
          const int n0 = (t0 + j) * BN;
          for (int kb = 0; kb < g.total_kb; ++kb) {
            const uint32_t dst = b_smem + s * THIN_B_STAGE + kb * 2 * B_TILE;
            const int b1 = B_MN ? kb * BK : n0, b2 = B_MN ? (n0 / BK) : kb;
            tma_load_3d(&pr.b_hi, fb, dst, 0, b1, b2);
            tma_load_3d(&pr.b_lo, fb, dst + B_TILE, 0, b1, b2);
          }
        }
      }
    }
    return;
  }

  // ================= math warpgroups =================
  const int wgi = warp >> 2, wq = warp & 3;
  const int gid = lane >> 2, tq = lane & 3;        // accumulator fragment coordinates
  const uint32_t stage = smem_u32(acc_stage + wgi * THIN_ACC_FLOATS);
  const uint32_t slab_hi = smem_u32(slabs) + (uint32_t)wgi * THIN_SLAB_WG, slab_lo = slab_hi + THIN_SLAB_WG / 2;
  const int srow = 32 * (wq >> 1) + lane, scol = 32 * (wq & 1);   // this warp's slice of the 64 x 64 unit
  int cur = 0, next0 = first_next0(grp);
  uint32_t tile = 0, icount = 0;                   // B tiles and items of this CTA so far (2 tile 64-row units)
  for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++icount) {
    cur = find_problem(grp, cur, item, next0);
    const Problem& pr = grp.p[cur];
    const GemmParams& g = pr.g;
    const int runs = thin_runs(g.tiles_n), local = item - pr.item0;
    const int mb = local / runs, t0 = (local - mb * runs) * THIN_RUN;
    const int nt = min(THIN_RUN, g.tiles_n - t0);
    // this warpgroup's units of the item: u0, u0 + THIN_WGS, ... < 2 nt
    const int u0 = (int)((wgi + THIN_WGS - 2 * tile % THIN_WGS) % THIN_WGS);
    mbar_wait(smem_u32(a_full), icount & 1u);
    if (u0 >= 2 * nt && lane == 0) mbar_arrive(smem_u32(a_empty));
    for (int u = u0; u < 2 * nt; u += THIN_WGS) {
      const int j = u >> 1, half = u & 1;
      const uint32_t t = tile + j, s = t % THIN_STAGES;
      const int n0 = (t0 + j) * BN;
      // dX: the ReLU-mask word of the lane's row, loaded before the MMAs (all ones without a mask, 0 past M)
      uint32_t mw = 0xffffffffu;
      if (EPI == EPI_MASK && g.mask_bits) {
        const int my_row = mb * BM + 64 * half + srow, kbo = (n0 + scol) >> 5;
        mw = (my_row < g.M && kbo < g.out_nb32) ? __ldg(g.mask_bits + (size_t)kbo * g.M + my_row) : 0u;
      }
      mbar_wait(smem_u32(&full_bar[s]), (t / THIN_STAGES) & 1u);
      // MMA accumulators of this unit only: nothing keeps them live through the epilogue (4 warps of a quadrant
      // share its registers at THIN_THREADS, so a thread has 128)
      float H[32], S[32];
#pragma unroll
      for (int jj = 0; jj < 32; ++jj) H[jj] = S[jj] = 0.f;
      wg::fence_regs(H);
      wg::fence_regs(S);
      wg::fence();
      const uint32_t a_st = a_smem + half * 8192u, b_st = b_smem + s * THIN_B_STAGE;
      f16_kblock_at<A_MN, B_MN>(a_st, b_st, H, S, true);
      if (g.total_kb > 1) f16_kblock_at<A_MN, B_MN>(a_st + 2 * A_TILE, b_st + 2 * B_TILE, H, S, false);
      wg::commit();
      wg::wait<0>();
      wg::fence_regs(H);
      wg::fence_regs(S);
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(smem_u32(&empty_bar[s]));
        if (u + THIN_WGS >= 2 * nt) mbar_arrive(smem_u32(a_empty));   // this warp's last MMA on the item's A rows
      }
      float acc[32];
      const int c0 = n0 + 2 * tq;
      const float* bias = (EPI == EPI_BIAS_ACT && g.bias) ? g.bias + c0 : nullptr;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e) {       // the bias starts the accumulation
          const int dc = 8 * jj + (e & 1);
          acc[4 * jj + e] = (bias && c0 + dc < g.N) ? __ldg(bias + dc) : 0.f;
        }
      fold_chunk<FMT_F16>(acc, H, S);
      // fragment layout -> staging area -> row per lane.  Past this barrier the warpgroup's previous slices have been
      // read, and its previous tile stores have read the slabs (the issuing thread waited for them).
      if (wq == 0 && lane == 0) bulk_wait_read0();
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wgi) : "memory");
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {   // 32-bit shared addresses: 64-bit generic ones for every store ran out of registers
        const int row = 16 * wq + gid, col = 8 * jj + 2 * tq;
        sts_v2(stage + 4u * acc_off(row, col), acc[4 * jj], acc[4 * jj + 1]);
        sts_v2(stage + 4u * acc_off(row + 8, col), acc[4 * jj + 2], acc[4 * jj + 3]);
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wgi) : "memory");
      float a[32];
#pragma unroll
      for (int q = 0; q < 8; ++q) lds_v4(stage + 4u * acc_off(srow, scol + 4 * q), a[4 * q], a[4 * q + 1], a[4 * q + 2], a[4 * q + 3]);
      // the lane's row of each plane goes into the warpgroup's [64 rows][128 B] slabs (16 B chunk ^= row % 8, the
      // SWIZZLE_128B layout); one thread then stores the 64 x 64 unit of each plane with a single TMA store, 128 B
      // per row, instead of four 32 x 32 boxes of 64 B rows per plane
      const auto store16 = [&](const float* v) {
        uint32_t w[16], lw[16];
        split_f16x32(v, w, lw);
        const uint32_t roff = (uint32_t)srow * 128u, sw = (uint32_t)srow & 7u, c0 = (uint32_t)scol >> 3;
#pragma unroll
        for (uint32_t q = 0; q < 4; ++q) {
          sts_v4(slab_hi + roff + (((c0 + q) ^ sw) << 4), w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
          sts_v4(slab_lo + roff + (((c0 + q) ^ sw) << 4), lw[4 * q], lw[4 * q + 1], lw[4 * q + 2], lw[4 * q + 3]);
        }
      };
      const int mrow0 = mb * BM + 64 * half + 32 * (wq >> 1), cbase = n0 + scol;
      if (EPI == EPI_BIAS_ACT) {
        const uint32_t drop_step = g.drop_thresh != 0u ? (uint32_t)(*g.drop_step) : 0u;
        emit_slice_fwd_planes<FMT_F16>(g, a, drop_step, lane, mrow0, cbase, nullptr, nullptr, 0u, 0u, &store16);
      }
      else
        emit_slice_mask_planes<FMT_F16>(g, a, mw, lane, mrow0, cbase, nullptr, nullptr, 0u, 0u, &store16);
      fence_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wgi) : "memory");
      if (wq == 0 && lane == 0) {
        tma_store_3d(&pr.o_hi, slab_hi, 0, mb * BM + 64 * half, n0 / BK);
        tma_store_3d(&pr.o_lo, slab_lo, 0, mb * BM + 64 * half, n0 / BK);
        bulk_commit();
      }
    }
    tile += nt;
  }
  if (wq == 0 && lane == 0) bulk_wait0();    // stores complete before the CTA (and its shared memory) goes away
}

// ---------------------------------------------------------------------------------
// dense <-> planes conversion (inputs x / labels-side gradients / weights; everything
// between two GEMMs is written as planes by the producing epilogue instead)
// ---------------------------------------------------------------------------------
// src[rows, cols] row-major (times `scale`, a power of two) -> hi/lo[nkb][rows][BK] (zero padded in cols) +
// sign bits[nkb * BK/32][rows]
template <int FMT>
__global__ void __launch_bounds__(256)
split_kernel(const float* __restrict__ src, void* __restrict__ hi_, void* __restrict__ lo_, uint32_t* __restrict__ bits,
             int rows, int cols, int nkb, float scale, unsigned int* ovf) {
  constexpr int BK = Fmt<FMT>::BK;
  const int vec_per_row = nkb * (BK / 4);                // float4 per padded row; 8 consecutive threads = one sign word
  const int64_t nvec = (int64_t)rows * vec_per_row;
  const int64_t nvec_pad = (nvec + 31) & ~(int64_t)31;   // whole warps run the loop (shuffles below)
  const bool vec_src = ((cols & 3) == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  bool over = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec_pad; i += (int64_t)gridDim.x * blockDim.x) {
    const bool live = i < nvec;
    const int r = live ? (int)(i / vec_per_row) : 0;
    const int c = live ? (int)(i % vec_per_row) * 4 : 0;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (live) {
      if (vec_src && c + 3 < cols) {
        float4 t = __ldg(reinterpret_cast<const float4*>(src + (size_t)r * cols + c));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = (c + q < cols) ? __ldg(src + (size_t)r * cols + c + q) : 0.f;
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) v[q] *= scale;
    }
    uint32_t nib = 0u;
#pragma unroll
    for (int q = 0; q < 4; ++q) nib |= (v[q] > 0.f) ? (1u << q) : 0u;
    uint32_t w = nib << (4 * (threadIdx.x & 7));
    w |= __shfl_xor_sync(0xffffffffu, w, 1);
    w |= __shfl_xor_sync(0xffffffffu, w, 2);
    w |= __shfl_xor_sync(0xffffffffu, w, 4);
    if (live) {
      const size_t dst = ((size_t)(c / BK) * rows + r) * BK + (c % BK);
      if (FMT == FMT_F16) {
        __half h[4], l[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          split_f16(v[q], h[q], l[q]);
          over |= f16_overflows(v[q]);
        }
        *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(hi_) + dst) = make_uint2(pack_h2(h[0], h[1]), pack_h2(h[2], h[3]));
        *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(lo_) + dst) = make_uint2(pack_h2(l[0], l[1]), pack_h2(l[2], l[3]));
      } else {
        float h[4], l[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) split_tf32(v[q], h[q], l[q]);
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(hi_) + dst) = make_float4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(lo_) + dst) = make_float4(l[0], l[1], l[2], l[3]);
      }
      if ((threadIdx.x & 7) == 0) bits[(size_t)(c >> 5) * rows + r] = w;
    }
  }
  if (over) raise_overflow(ovf);
}

// hi/lo[nkb][rows][BK] -> dst[rows, cols] = hi + lo (tf32) | hi + 2^-11 lo' (f16)
template <int FMT>
__global__ void __launch_bounds__(256)
merge_kernel(const void* __restrict__ hi_, const void* __restrict__ lo_, float* __restrict__ dst, int rows, int cols, int nkb) {
  constexpr int BK = Fmt<FMT>::BK;
  const int64_t n = (int64_t)rows * nkb * BK;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cb = (int)(i % BK);
    const int64_t t = i / BK;
    const int r = (int)(t % rows);
    const int c = (int)(t / rows) * BK + cb;
    if (c < cols) {
      if (FMT == FMT_F16)
        dst[(size_t)r * cols + c] = merge_f16(reinterpret_cast<const __half*>(hi_)[i], reinterpret_cast<const __half*>(lo_)[i]);
      else
        dst[(size_t)r * cols + c] = reinterpret_cast<const float*>(hi_)[i] + reinterpret_cast<const float*>(lo_)[i];
    }
  }
}

// ---------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------
__device__ unsigned int g_plane_overflow = 0u;

static PFN_cuTensorMapEncodeTiled g_encode = nullptr;
static unsigned int* g_ovf_addr = nullptr;
static std::atomic<int> g_format{-1};

int format() {
  int f = g_format.load();
  if (f >= 0) return f;
  const char* e = getenv("ADN_PLANES");
  f = (e && (!strcmp(e, "tf32") || !strcmp(e, "TF32"))) ? FMT_TF32 : FMT_F16;
  g_format.store(f);
  return f;
}
int set_format(int fmt) {
  if (fmt != FMT_TF32 && fmt != FMT_F16) return fail(ADN_ERR_INVALID, "adn_set_plane_format: bad format %d", fmt);
  g_format.store(fmt);
  return ADN_OK;
}
unsigned int* overflow_flag() { return g_ovf_addr; }

int read_overflow(int* out_host, int reset, cudaStream_t st) {
  if (!g_ovf_addr) return fail(ADN_ERR_CUDA, "pl: adn_init() was not called");
  unsigned int v = 0;
  ADN_CUDA(cudaMemcpyAsync(&v, g_ovf_addr, sizeof(v), cudaMemcpyDeviceToHost, st));
  if (reset) ADN_CUDA(cudaMemsetAsync(g_ovf_addr, 0, sizeof(v), st));
  ADN_CUDA(cudaStreamSynchronize(st));
  *out_host = (int)v;
  return ADN_OK;
}

int init() {
  static std::once_flag once;
  static int rc = ADN_OK;
  std::call_once(once, []() {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || fn == nullptr) {
      (void)cudaGetLastError();
      rc = fail(ADN_ERR_CUDA, "pl::init: cuTensorMapEncodeTiled entry point unavailable");
      return;
    }
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(fn);
    bool ok = true;
#define ADN_PL_ATTR(F, E) \
  ok = ok && (cudaFuncSetAttribute(pl_gemm_kernel<F, E>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) == cudaSuccess)
    ADN_PL_ATTR(FMT_TF32, EPI_BIAS_ACT); ADN_PL_ATTR(FMT_TF32, EPI_MASK); ADN_PL_ATTR(FMT_TF32, EPI_PARTIAL);
    ADN_PL_ATTR(FMT_F16, EPI_BIAS_ACT); ADN_PL_ATTR(FMT_F16, EPI_MASK); ADN_PL_ATTR(FMT_F16, EPI_PARTIAL);
#undef ADN_PL_ATTR
    ok = ok && cudaFuncSetAttribute(pl_gemm_ms_kernel<FMT_TF32>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(pl_gemm_ms_kernel<FMT_F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(pl_thin_kernel<EPI_BIAS_ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, THIN_SMEM_BYTES) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(pl_thin_kernel<EPI_MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, THIN_SMEM_BYTES) == cudaSuccess;
    if (!ok) {
      (void)cudaGetLastError();
      rc = fail(ADN_ERR_CUDA, "pl::init: cudaFuncSetAttribute(smem=%d) failed", SMEM_BYTES);
      return;
    }
    void* addr = nullptr;
    if (cudaGetSymbolAddress(&addr, g_plane_overflow) != cudaSuccess || !addr) {
      (void)cudaGetLastError();
      rc = fail(ADN_ERR_CUDA, "pl::init: cudaGetSymbolAddress(g_plane_overflow) failed");
      return;
    }
    g_ovf_addr = reinterpret_cast<unsigned int*>(addr);
  });
  return rc;
}

int64_t planes_bytes_fmt(int fmt, int64_t rows, int64_t cols) { return planes_bytes(fmt, rows, cols); }

// a plane tensor viewed as a GEMM operand
struct Operand {
  const void* hi;
  const void* lo;
  int64_t rows, nkb;
  int mn_major;
};
static Operand operand(int fmt, const void* planes, int64_t rows, int64_t cols, int mn_major) {
  const char* p = reinterpret_cast<const char*>(planes);
  return Operand{p, p + plane_bytes1(fmt, rows, cols), rows, ceil_div(cols, fmt_bk(fmt)), mn_major};
}

// ---- TMA descriptor cache (include/adanet_b200.h conventions): a descriptor depends only on (plane base, rows,
// k-blocks, majorness, tile extent, format); the same few hundred recur on every eager step, eval pass and graph
// re-capture.
struct MapKey {
  const void* ptr;
  int64_t rows, nkb;
  int mn, fmt;
  int box = 0;           // tile extent of the operand (BM for A, BN for B); 0 for the store boxes
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && rows == o.rows && nkb == o.nkb && mn == o.mn && fmt == o.fmt && box == o.box;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<uintptr_t>(k.ptr) * 0x9E3779B97F4A7C15ull;
    h ^= (size_t)k.rows * 0xC2B2AE3D27D4EB4Full + ((size_t)k.nkb << 20) + ((size_t)k.mn << 1) + (size_t)k.fmt + ((size_t)k.box << 40);
    return h ^ (h >> 29);
  }
};
static std::mutex g_map_mu;
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
static std::atomic<long long> g_map_hits{0}, g_map_misses{0};
long long map_cache_hits() { return g_map_hits.load(); }
long long map_cache_misses() { return g_map_misses.load(); }

// operand tile of `box` rows (K-major) or columns (MN-major) per k-block
static int make_map(int fmt, CUtensorMap* map, const void* plane, int64_t rows, int64_t nkb, int mn_major, int box) {
  if (!g_encode) return fail(ADN_ERR_CUDA, "pl: adn_init() was not called");
  const MapKey key{plane, rows, nkb, mn_major, fmt, box};
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) {
      *map = it->second;
      g_map_hits.fetch_add(1, std::memory_order_relaxed);
      return ADN_OK;
    }
  }
  const int bk = fmt_bk(fmt), es = fmt_esize(fmt);
  cuuint64_t gdim[3] = {(cuuint64_t)bk, (cuuint64_t)rows, (cuuint64_t)nkb};
  cuuint64_t gstride[2] = {(cuuint64_t)bk * es, (cuuint64_t)rows * bk * es};
  cuuint32_t box_k[3] = {(cuuint32_t)bk, (cuuint32_t)box, 1u};
  cuuint32_t box_mn[3] = {(cuuint32_t)bk, (cuuint32_t)bk, (cuuint32_t)(box / bk)};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = g_encode(map, fmt == FMT_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3,
                        const_cast<void*>(plane), gdim, gstride, mn_major ? box_mn : box_k, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(ADN_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%lld nkb=%lld mn=%d fmt=%d", (int)r,
                                     (long long)rows, (long long)nkb, mn_major, fmt);
  g_map_misses.fetch_add(1, std::memory_order_relaxed);
  std::lock_guard<std::mutex> lk(g_map_mu);
  if (g_maps.size() > 16384) g_maps.clear();     // bounded: buffers come and go with plans
  g_maps.emplace(key, *map);
  return ADN_OK;
}

// output planes (fp16) as TMA store targets: [box columns][box rows] boxes; box = 32 (pl_gemm_kernel's 32 x 32 slices,
// 64 B rows, SWIZZLE_64B in shared memory) or 64 (pl_thin_kernel's 64 x 64 units, 128 B rows, SWIZZLE_128B)
static int make_store_map(CUtensorMap* map, const void* plane, int64_t rows, int64_t nkb, int box_rc = 32) {
  if (!g_encode) return fail(ADN_ERR_CUDA, "pl: adn_init() was not called");
  const MapKey key{plane, rows, nkb, 2, FMT_F16, box_rc};      // mn = 2: a store box
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) {
      *map = it->second;
      g_map_hits.fetch_add(1, std::memory_order_relaxed);
      return ADN_OK;
    }
  }
  cuuint64_t gdim[3] = {64u, (cuuint64_t)rows, (cuuint64_t)nkb};
  cuuint64_t gstride[2] = {128u, (cuuint64_t)rows * 128u};
  cuuint32_t box[3] = {(cuuint32_t)box_rc, (cuuint32_t)box_rc, 1u};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(plane), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, box_rc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                        CU_TENSOR_MAP_L2_PROMOTION_NONE,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(ADN_ERR_CUDA, "cuTensorMapEncodeTiled (store box) failed (%d) rows=%lld nkb=%lld", (int)r,
                                     (long long)rows, (long long)nkb);
  g_map_misses.fetch_add(1, std::memory_order_relaxed);
  std::lock_guard<std::mutex> lk(g_map_mu);
  if (g_maps.size() > 16384) g_maps.clear();
  g_maps.emplace(key, *map);
  return ADN_OK;
}
// one GEMM of a group: operands + epilogue description (tiles / item numbering are filled at launch)
struct GemmDesc {
  Operand a, b;
  GemmParams g;
  int n_src = 0;                       // multi-source forward: pieces (x, w) besides (a, b)
  Operand sa[MAX_SRCS], sb[MAX_SRCS];
};

static int encode_maps(int fmt, const GemmDesc& d, CUtensorMap* a_hi, CUtensorMap* a_lo, CUtensorMap* b_hi, CUtensorMap* b_lo,
                       const char* what) {
  if (!planes_aligned(d.a.hi) || !planes_aligned(d.a.lo) || !planes_aligned(d.b.hi) || !planes_aligned(d.b.lo))
    return fail(ADN_ERR_INVALID, "%s: plane buffers must be 256 B aligned", what);
  int rc;
  if ((rc = make_map(fmt, a_hi, d.a.hi, d.a.rows, d.a.nkb, d.a.mn_major, BM))) return rc;
  if ((rc = make_map(fmt, a_lo, d.a.lo, d.a.rows, d.a.nkb, d.a.mn_major, BM))) return rc;
  if ((rc = make_map(fmt, b_hi, d.b.hi, d.b.rows, d.b.nkb, d.b.mn_major, BN))) return rc;
  if ((rc = make_map(fmt, b_lo, d.b.lo, d.b.rows, d.b.nkb, d.b.mn_major, BN))) return rc;
  return ADN_OK;
}

// A group runs on pl_thin_kernel when every problem is one fp16 accumulation chunk with planes out and no split.
static bool thin_group(int fmt, const Group& grp) {
  if (fmt != FMT_F16) return false;
  for (int i = 0; i < grp.n; ++i) {
    const GemmParams& g = grp.p[i].g;
    if (!g.out_planes || g.splits != 1 || g.total_kb > Fmt<FMT_F16>::CHUNK) return false;
  }
  return true;
}
template <int FMT, int EPI>
static void launch_kernel(const Group& grp, int grid, cudaStream_t st) {
  pl_gemm_kernel<FMT, EPI><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(grp);
}
// n independent GEMMs of the same epilogue kind -> parameter blocks of up to MAX_GROUP problems each, one per
// persistent launch (G = MsGroup: multi-source forward GEMMs, on pl_gemm_ms_kernel).  Every descriptor is encoded
// here, before anything is launched, so that a failure leaves every output as it was.
template <int EPI, class G>
static int build_groups(int fmt, const GemmDesc* d, int n, std::vector<G>& out, const char* what) {
  constexpr bool MS = std::is_same<G, MsGroup>::value;
  static_assert(!MS || EPI == EPI_BIAS_ACT, "multi-source GEMMs are forward only");
  out.clear();
  {
    for (int i0 = 0; i0 < n; i0 += MAX_GROUP) {
      const int m = std::min(MAX_GROUP, n - i0);
      out.emplace_back();
      G& grp = out.back();
      memset(&grp, 0, sizeof(grp));
      int items = 0;
      for (int i = 0; i < m; ++i) {
        const GemmDesc& src = d[i0 + i];
        auto& pr = grp.p[i];
        // the kernel fixes the operand majorness per epilogue kind (fwd: K / MN, dX: K / K, dW: MN / MN)
        if (src.a.mn_major != (EPI == EPI_PARTIAL) || src.b.mn_major != (EPI != EPI_MASK))
          return fail(ADN_ERR_INVALID, "%s: operand majorness does not match the epilogue kind", what);
        int rc = encode_maps(fmt, src, &pr.a_hi, &pr.a_lo, &pr.b_hi, &pr.b_lo, what);
        if (rc) return rc;
        if constexpr (MS) {
          int kb = (int)src.a.nkb;
          pr.n_src = src.n_src;
          pr.kb_end[0] = kb;
          for (int q = 0; q < src.n_src; ++q) {
            GemmDesc piece;
            piece.a = src.sa[q];
            piece.b = src.sb[q];
            if ((rc = encode_maps(fmt, piece, &pr.src[q][0], &pr.src[q][1], &pr.src[q][2], &pr.src[q][3], what))) return rc;
            kb += (int)src.sa[q].nkb;
            pr.kb_end[q + 1] = kb;
          }
          if (kb != src.g.total_kb) return fail(ADN_ERR_INVALID, "%s: k-blocks of the pieces do not add up", what);
        }
        pr.g = src.g;
        // fp16 plane tiles leave the epilogue by TMA stores (the API checked yp / dxp against planes_aligned)
        if (fmt == FMT_F16 && src.g.out_planes) {
          if ((rc = make_store_map(&pr.o_hi, src.g.out, src.g.M, src.g.out_nb32 / 2))) return rc;
          if ((rc = make_store_map(&pr.o_lo, src.g.out_lo, src.g.M, src.g.out_nb32 / 2))) return rc;
        }
        pr.g.a_mn = src.a.mn_major;
        pr.g.b_mn = src.b.mn_major;
        pr.g.tiles_m = (int)ceil_div(pr.g.M, BM);
        pr.g.tiles_n = (int)ceil_div(pr.g.N, BN);
        pr.g.tiles = pr.g.tiles_m * pr.g.tiles_n;
        if ((int64_t)pr.g.tiles * pr.g.splits >= (1 << 21))
          return fail(ADN_ERR_UNSUPPORTED, "%s: %d work items exceed the decode range", what, pr.g.tiles * pr.g.splits);
        pr.g.inv_tiles = 1.0f / (float)pr.g.tiles;
        pr.g.inv_tiles_n = 1.0f / (float)pr.g.tiles_n;
        pr.g.ovf = g_ovf_addr;
        pr.item0 = items;
        items += pr.g.tiles_m * pr.g.tiles_n * pr.g.splits;
      }
      grp.n = m;
      grp.total_items = items;
      if constexpr (!MS) {
        if (thin_group(fmt, grp)) {     // pl_thin_kernel's work items (128-row block x run of THIN_RUN N tiles) and store boxes
          items = 0;
          for (int i = 0; i < m; ++i) {
            Problem& pr = grp.p[i];
            pr.item0 = items;
            items += pr.g.tiles_m * thin_runs(pr.g.tiles_n);
            int rc;
            if ((rc = make_store_map(&pr.o_hi, pr.g.out, pr.g.M, pr.g.out_nb32 / 2, 64))) return rc;
            if ((rc = make_store_map(&pr.o_lo, pr.g.out_lo, pr.g.M, pr.g.out_nb32 / 2, 64))) return rc;
          }
          grp.total_items = items;
        }
      }
    }
  }
  return ADN_OK;
}
template <int EPI, class G>
static int launch_groups(int fmt, const std::vector<G>& groups, cudaStream_t st, const char* what) {
  for (const G& grp : groups) {
    const int grid = std::min(grp.total_items, sm_count());
    if constexpr (std::is_same<G, MsGroup>::value) {
      if (fmt == FMT_F16) pl_gemm_ms_kernel<FMT_F16><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(grp);
      else pl_gemm_ms_kernel<FMT_TF32><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(grp);
    } else if (thin_group(fmt, grp)) {
      if constexpr (EPI != EPI_PARTIAL) pl_thin_kernel<EPI><<<grid, THIN_THREADS, THIN_SMEM_BYTES, st>>>(grp);
    } else {
      if (fmt == FMT_F16) launch_kernel<FMT_F16, EPI>(grp, grid, st);
      else launch_kernel<FMT_TF32, EPI>(grp, grid, st);
    }
    ADN_CHECK_LAUNCH(what);
  }
  return ADN_OK;
}
template <int EPI>
static int launch_group(int fmt, const GemmDesc* d, int n, cudaStream_t st, const char* what) {
  std::vector<Group> groups;
  const int rc = build_groups<EPI>(fmt, d, n, groups, what);
  return rc ? rc : launch_groups<EPI>(fmt, groups, st, what);
}

int split(int fmt, const float* src, int64_t rows, int64_t cols, void* planes, int log2_scale, cudaStream_t st) {
  const int bk = fmt_bk(fmt);
  const int64_t nkb = ceil_div(cols, bk);
  const int64_t nvec = rows * nkb * (bk / 4);
  const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(nvec, 256), (int64_t)sm_count() * 16));
  const PlaneView v = plane_view(fmt, planes, rows, cols);
  const float scale = ldexpf(1.0f, log2_scale);
  if (fmt == FMT_F16)
    split_kernel<FMT_F16><<<blocks, 256, 0, st>>>(src, v.hi, v.lo, v.bits, (int)rows, (int)cols, (int)nkb, scale, g_ovf_addr);
  else
    split_kernel<FMT_TF32><<<blocks, 256, 0, st>>>(src, v.hi, v.lo, v.bits, (int)rows, (int)cols, (int)nkb, scale, g_ovf_addr);
  ADN_CHECK_LAUNCH("planes split");
  return ADN_OK;
}

int merge(int fmt, const void* planes, int64_t rows, int64_t cols, float* dst, cudaStream_t st) {
  const int bk = fmt_bk(fmt);
  const int64_t nkb = ceil_div(cols, bk);
  const int64_t n = rows * nkb * bk;
  const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256), (int64_t)sm_count() * 16));
  const PlaneView v = plane_view(fmt, const_cast<void*>(planes), rows, cols);
  if (fmt == FMT_F16) merge_kernel<FMT_F16><<<blocks, 256, 0, st>>>(v.hi, v.lo, dst, (int)rows, (int)cols, (int)nkb);
  else merge_kernel<FMT_TF32><<<blocks, 256, 0, st>>>(v.hi, v.lo, dst, (int)rows, (int)cols, (int)nkb);
  ADN_CHECK_LAUNCH("planes merge");
  return ADN_OK;
}

// dW split-K: the partial buffer bounds the split count (<= 16M floats, <= 64 splits)
static int max_dw_splits(int64_t in, int64_t out) {
  int64_t s = (16LL << 20) / std::max<int64_t>(1, in * out);
  if (s > MAX_SPLITS) s = MAX_SPLITS;
  if (s < 1) s = 1;
  return (int)s;
}

int64_t dense_bwd_workspace_bytes(int64_t batch, int64_t in, int64_t out) {
  int64_t b = align_up((int64_t)max_dw_splits(in, out) * in * out * (int64_t)sizeof(float), 256);   // dW split-K partials
  b += align_up(ceil_div(batch, 32) * in * (int64_t)sizeof(float), 256);                             // dx column sums per 32 rows
  b += align_up(64 * in * (int64_t)sizeof(float), 256);                                              // their second-level partials
  return b + 512;
}

int dense_fwd_group(int fmt, const FwdOp* ops, int n, int64_t batch, cudaStream_t st) {
  if (n <= 0) return ADN_OK;
  const int bk = fmt_bk(fmt);
  std::vector<GemmDesc> d, dm;     // single-source ops, multi-source ops
  d.reserve((size_t)n);
  for (int i = 0; i < n; ++i) {
    const FwdOp& o = ops[i];
    GemmDesc e;
    e.a = operand(fmt, o.xp, batch, o.in, 0);       // A = x  [M=batch, K=in]  K-major
    e.b = operand(fmt, o.wp, o.in, o.out, 1);       // B = w  [K=in, N=out]    MN-major
    int64_t kb = ceil_div(o.in, bk);
    e.n_src = o.n_srcs;
    for (int q = 0; q < o.n_srcs; ++q) {             // piece q: x_q [batch, in_q] times rows of w [in_q, out]
      e.sa[q] = operand(fmt, o.srcs[q].xp, batch, o.srcs[q].in, 0);
      e.sb[q] = operand(fmt, o.srcs[q].wp, o.srcs[q].in, o.out, 1);
      kb += ceil_div(o.srcs[q].in, bk);
    }
    GemmParams g{};
    g.M = (int)batch; g.N = (int)o.out;
    g.total_kb = (int)kb; g.kb_per_split = g.total_kb; g.splits = 1;
    g.bias = o.bias; g.act = o.act;
    g.out_mul = 1.0f;
    if (o.dropout_rate > 0.f) {
      if (!o.yp || !o.dropout_step) return fail(ADN_ERR_INVALID, "pl dense_fwd: dropout needs planes out and a step counter");
      const double t = (double)o.dropout_rate * 4294967296.0;
      g.drop_thresh = t >= 4294967295.0 ? 0xffffffffu : (uint32_t)t;
      if (g.drop_thresh == 0u) g.drop_thresh = 1u;
      g.drop_key0 = o.dropout_seed * 0x9E3779B1u + (uint32_t)o.dropout_layer * 0x85EBCA77u + 0x27D4EB2Fu;
      g.drop_scale = 1.0f / (1.0f - o.dropout_rate);
      g.drop_idx0 = (uint32_t)((uint64_t)o.dropout_row0 * (uint64_t)o.out);
      g.drop_step = o.dropout_step;
    }
    if (o.yp) {
      const PlaneView v = plane_view(fmt, o.yp, batch, o.out);
      g.out_planes = 1;
      g.out = v.hi; g.out_lo = v.lo; g.out_nb32 = (int)bits_blocks(fmt, o.out);
      g.out_bits = v.bits;
    } else {
      g.out = o.y; g.ldc = (int)o.out;
    }
    e.g = g;
    (o.n_srcs ? dm : d).push_back(e);
  }
  // both kinds are encoded before either is launched: a call that returns an error has written nothing
  std::vector<Group> groups;
  std::vector<MsGroup> ms_groups;
  int rc;
  if ((rc = build_groups<EPI_BIAS_ACT>(fmt, d.data(), (int)d.size(), groups, "pl dense_fwd gemm"))) return rc;
  if ((rc = build_groups<EPI_BIAS_ACT>(fmt, dm.data(), (int)dm.size(), ms_groups, "pl dense_fwd multi-source gemm"))) return rc;
  if ((rc = launch_groups<EPI_BIAS_ACT>(fmt, groups, st, "pl dense_fwd gemm"))) return rc;
  return launch_groups<EPI_BIAS_ACT>(fmt, ms_groups, st, "pl dense_fwd multi-source gemm");
}

int dense_bwd_group(int fmt, const BwdOp* ops, int n, int64_t batch, cudaStream_t st) {
  if (n <= 0) return ADN_OK;
  const int bk = fmt_bk(fmt);
  const int workers = sm_count();
  struct Carve { float* part; float* cspart; float* cspart2; int splits; };
  std::vector<Carve> cv((size_t)n);
  std::vector<GemmDesc> dwd, dxd;
  // Split-K over the batch for the dW GEMMs of the group.  Work items of one launch are dealt round-robin to the
  // CTAs (item j -> CTA j % grid), so the launch takes as long as its most loaded CTA.  Every problem uses the
  // k-blocks-per-item `kps` (raised to its own partial-buffer bound), and kps is chosen by evaluating, for every
  // candidate split count, the exact round-robin load (k-blocks + a per-item pipeline fill/drain + epilogue
  // allowance) plus the cost of the fixed-order reduction of the partial sums (bytes at ~2.5 TB/s; one k-block
  // of MMA work is ~0.4 us).  (A k-block is 4 MMA steps in either format.)
  const int64_t kb_b = ceil_div(batch, bk);
  int64_t best_kps = kb_b;
  {
    static std::mutex mu;
    static std::unordered_map<std::string, int64_t> memo;      // the same waves recur every step / capture
    std::string key = std::to_string(batch) + ":" + std::to_string(fmt);
    for (int i = 0; i < n; ++i)
      if (ops[i].dw) key += "," + std::to_string(ops[i].in) + "x" + std::to_string(ops[i].out);
    bool hit = false;
    {
      std::lock_guard<std::mutex> lk(mu);
      auto it = memo.find(key);
      if (it != memo.end()) { best_kps = it->second; hit = true; }
    }
    if (!hit) {
      const double kItemOverhead = 6.0;          // k-block equivalents per work item
      const double kReduceKbPerByte = 1.0 / (2.5e6 * 0.4);     // k-block equivalents per byte of partials read
      double best_t = 1e30;
      std::vector<double> load((size_t)workers);
      int64_t last_kps = -1;
      for (int s0 = 1; s0 <= MAX_SPLITS && s0 <= kb_b; ++s0) {
        const int64_t kps = ceil_div(kb_b, s0);
        if (kps == last_kps) continue;
        last_kps = kps;
        std::fill(load.begin(), load.end(), 0.0);
        int64_t item = 0;
        double reduce_bytes = 0.0;
        bool any = false;
        for (int i = 0; i < n; ++i) {
          if (!ops[i].dw) continue;
          any = true;
          const int64_t k_i = std::max<int64_t>(kps, ceil_div(kb_b, max_dw_splits(ops[i].in, ops[i].out)));
          const int64_t s_i = ceil_div(kb_b, k_i);
          const int64_t tiles = ceil_div(ops[i].in, BM) * ceil_div(ops[i].out, BN);
          for (int64_t sp = 0; sp < s_i; ++sp) {
            const double kb_item = (double)(std::min(kb_b, (sp + 1) * k_i) - sp * k_i);
            for (int64_t t = 0; t < tiles; ++t, ++item) load[(size_t)(item % workers)] += kb_item + kItemOverhead;
          }
          if (s_i > 1) reduce_bytes += (double)(s_i + 1) * (double)ops[i].in * (double)ops[i].out * 4.0;
        }
        if (!any) break;
        const double t = *std::max_element(load.begin(), load.end()) +
                         reduce_bytes * kReduceKbPerByte + (reduce_bytes > 0 ? 10.0 : 0.0);
        if (t < best_t) { best_t = t; best_kps = kps; }
      }
      std::lock_guard<std::mutex> lk(mu);
      if (memo.size() > 4096) memo.clear();
      memo[key] = best_kps;
    }
  }
  for (int i = 0; i < n; ++i) {
    const BwdOp& o = ops[i];
    if (!o.ws || o.ws_bytes < dense_bwd_workspace_bytes(batch, o.in, o.out))
      return fail(ADN_ERR_WORKSPACE, "pl dense_bwd: op %d workspace %lld < %lld bytes", i, (long long)o.ws_bytes,
                  (long long)dense_bwd_workspace_bytes(batch, o.in, o.out));
    const float unscale = ldexpf(1.0f, -o.dz_log2_scale);
    char* p = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(o.ws) + 255) & ~(uintptr_t)255);
    const int max_s = max_dw_splits(o.in, o.out);
    Carve& c = cv[(size_t)i];
    c.part = reinterpret_cast<float*>(p);
    p += align_up((int64_t)max_s * o.in * o.out * (int64_t)sizeof(float), 256);
    c.cspart = reinterpret_cast<float*>(p);
    p += align_up(ceil_div(batch, 32) * o.in * (int64_t)sizeof(float), 256);
    c.cspart2 = reinterpret_cast<float*>(p);
    c.splits = 1;
    if (o.dw) {
      // ---- dW[in,out] = X^T dZ : A = Xp MN-major (M=in), B = dZp MN-major (N=out), K = batch, split-K ----
      GemmDesc e;
      e.a = operand(fmt, o.xp, batch, o.in, 1);
      e.b = operand(fmt, o.dzp, batch, o.out, 1);
      GemmParams g{};
      g.M = (int)o.in; g.N = (int)o.out; g.ldc = (int)o.out;
      g.total_kb = (int)kb_b; g.kb_per_split = (int)std::max<int64_t>(best_kps, ceil_div(kb_b, max_s));
      g.splits = (int)ceil_div(kb_b, g.kb_per_split);
      g.out = (g.splits == 1) ? o.dw : c.part;
      g.out_mul = (g.splits == 1) ? unscale : 1.0f;      // partials are un-scaled by the fixed-order reduction
      c.splits = g.splits;
      e.g = g;
      dwd.push_back(e);
    }
    if (o.dxp || o.dx) {
      // ---- dX[batch,in] = dZ W^T : A = dZp K-major (K=out), B = Wp K-major (N=in, K=out); ReLU mask = sign bits of X ----
      GemmDesc e;
      e.a = operand(fmt, o.dzp, batch, o.out, 0);
      e.b = operand(fmt, o.wp, o.in, o.out, 0);
      GemmParams g{};
      g.M = (int)batch; g.N = (int)o.in;
      g.total_kb = (int)ceil_div(o.out, bk); g.kb_per_split = g.total_kb; g.splits = 1;
      g.mask_bits = o.x_relu_mask ? bits_of(fmt, o.xp, batch, o.in) : nullptr;
      g.out_nb32 = (int)bits_blocks(fmt, o.in);
      g.colsum_part = o.dx_colsum ? c.cspart : nullptr;
      g.colsum_ld = (int)o.in;
      if (o.dxp) {
        const PlaneView v = plane_view(fmt, o.dxp, batch, o.in);
        g.out_planes = 1;
        g.out = v.hi; g.out_lo = v.lo;
        g.out_mul = o.dx_mul;              // the gradient keeps its scale while it stays in plane format
      } else {
        g.out = o.dx; g.ldc = (int)o.in;
        g.out_mul = unscale * o.dx_mul;    // dense fp32 leaves the plane pipeline: true magnitude
      }
      e.g = g;
      dxd.push_back(e);
    }
  }
  int rc;
  if (!dwd.empty()) {
    if ((rc = launch_group<EPI_PARTIAL>(fmt, dwd.data(), (int)dwd.size(), st, "pl dW gemm"))) return rc;
    std::vector<simt::ReduceJob> jobs;
    for (int i = 0; i < n; ++i)
      if (ops[i].dw && cv[(size_t)i].splits > 1)
        jobs.push_back(simt::ReduceJob{cv[(size_t)i].part, ops[i].dw, ops[i].in * ops[i].out, cv[(size_t)i].splits,
                                       ops[i].in * ops[i].out, ldexpf(1.0f, -ops[i].dz_log2_scale)});
    if ((rc = simt::reduce_partials_group(jobs.data(), (int)jobs.size(), st))) return rc;
  }
  if (!dxd.empty()) {
    if ((rc = launch_group<EPI_MASK>(fmt, dxd.data(), (int)dxd.size(), st, "pl dX gemm"))) return rc;
    // column sums of each [ceil(batch/32), in] partial matrix, fixed order
    std::vector<simt::ColsumJob> jobs;
    for (int i = 0; i < n; ++i)
      if (ops[i].dx_colsum && (ops[i].dxp || ops[i].dx))
        jobs.push_back(simt::ColsumJob{cv[(size_t)i].cspart, ops[i].dx_colsum, ceil_div(batch, 32), ops[i].in,
                                       cv[(size_t)i].cspart2, ops[i].dxp ? ldexpf(1.0f, -ops[i].dz_log2_scale) : 1.0f});
    if ((rc = simt::colsum_group(jobs.data(), (int)jobs.size(), st))) return rc;
  }
  return ADN_OK;
}

int dense_fwd(int fmt, const void* xp, const void* wp, const float* bias, void* yp, float* y, int64_t batch, int64_t in,
              int64_t out, int act, cudaStream_t st) {
  FwdOp op{xp, wp, bias, yp, y, in, out, act};
  return dense_fwd_group(fmt, &op, 1, batch, st);
}

int dense_bwd(int fmt, const void* xp, const void* wp, const void* dzp, void* dxp, float* dx, float* dx_colsum, float* dw,
              int64_t batch, int64_t in, int64_t out, int x_relu_mask, int dz_log2_scale, void* ws, int64_t ws_bytes,
              cudaStream_t st) {
  BwdOp op{xp, wp, dzp, dxp, dx, dx_colsum, dw, in, out, x_relu_mask, dz_log2_scale, ws, ws_bytes};
  return dense_bwd_group(fmt, &op, 1, batch, st);
}

}  // namespace pl
}  // namespace adn
