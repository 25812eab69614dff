// K6b: the SimpleCNN stem forward as a wgmma implicit GEMM (same contract as conv_stem_fwd_kernel in
// conv_stem.cu, which stays as the exact-fp32 cross-check path: ADN_CONV_PATH=simt).
//
// Formulation: rows = POOLED pixels, not conv positions.  For one pooled pixel the four conv positions of its 2x2
// window read a 4x4xCin input patch, so
//     acc[p][(pos, f)] = sum_k A[p][k] * W'[k][(pos, f)],   k = (i, j, c) over the 4x4xCin patch (K = 16*Cin),
//     W'[(i,j,c)][(dy,dx,f)] = w[i-dy][j-dx][c][f]  (zero outside the 3x3 support),   N = 4*F,
// is a [128 x K] x [K x N] GEMM per 128 pooled pixels whose accumulator row holds exactly what the epilogue thread
// of the SIMT kernel holds in registers: 4 positions x F filters of its own pooled pixel.  A thread of the wgmma
// accumulator layout holds the 4 positions of the same filters, so bias, ReLU, the 2x2 max and the arg-max stay in
// the thread; sign-bit and arg-max words are OR-ed over the 4 threads of a row.  The price is 1.78x the minimal MACs
// (zeros in W'), irrelevant at 3 x 6 wgmma (M64 N64 K8) per 64 pooled pixels.
//
// fp32 accuracy: 3xTF32 (a_hi b_hi + a_lo b_hi + a_hi b_lo), K <= 48, one accumulator.
//
// Per CTA (256 threads = 2 warpgroups, 1 CTA per SM): the image is staged zero-padded in shared memory with
// cp.async (double buffered); each warpgroup takes a tile of 128 pooled pixels: every thread gathers its own A row
// from the staged image (LDS.64), splits it and writes hi / lo in the canonical K-major SWIZZLE_128B layout
// (16-byte chunk index XOR row%8 -- what TMA would have produced), fence.proxy.async, then the warpgroup issues
// the MMAs of each 64-row half and runs the epilogue on the registers they return.  W' (hi / lo, K-major) is built
// once per CTA.
#include "common.cuh"
#include "plane_fmt.cuh"
#include "wgmma.cuh"

namespace adn {
namespace convtc {

static constexpr int THREADS = 256;
static constexpr int TILE_BYTES = 128 * 128;   // one k-block (32 floats) of a 128-row K-major SWIZZLE_128B tile

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wg_barrier(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }
// byte offset of element (row, k) inside one k-block tile ([rows][32 floats], SWIZZLE_128B)
__device__ __forceinline__ uint32_t sw128(int row, int k) {
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 2) ^ (row & 7)) & 7) << 4) + ((k & 3) << 2));
}
// D (+)= A B over one K step of 8, tf32, both operands K-major SWIZZLE_128B tiles in shared memory
template <int N>
__device__ __forceinline__ void mma_tf32(float (&d)[N / 2], uint32_t a_addr, uint32_t b_addr, uint32_t scale_d) {
  const uint64_t da = wg::desc_sw128(a_addr), db = wg::desc_sw128(b_addr);
  if constexpr (N == 64) wg::mma_tf32_n64(d, da, db, scale_d);
  else wg::mma_tf32_n128(d, da, db, scale_d);
}

template <int CIN>
__device__ __forceinline__ void stage_image(float* s_img, const float* img, int H, int W, int tid, int nthreads = THREADS) {
  const int row = W * CIN;
  const int prow = (W + 2) * CIN;
  const int lane = tid & 31;
  for (int y = tid >> 5; y < H; y += nthreads / 32) {
    const float* src = img + y * row;
    float* dst = s_img + (y + 1) * prow + CIN;
    for (int r = lane; r < row; r += 32) cp_async4(dst + r, src + r);
  }
}

// staged-image ring depth of the forward: 4 where shared memory allows (F = 16), else 2
__host__ __device__ constexpr int fwd_image_buffers(int f) { return f == 16 ? 4 : 2; }

// Forward.  256 threads = 2 warpgroups; warpgroup s takes the tiles s, s + 2, ... of every image: gather / split /
// swizzle the A rows of the tile, then per 64-row half issue the 3 x K/8 MMAs, wait, and run bias / ReLU / pool /
// split / store on the returned accumulators.
// Shared memory (from a 1024-aligned base): W' hi|lo [2][KB][N][128 B]; A per warpgroup hi|lo [2][KB][16 KB]; the
// ring of padded images; bias.
template <int CIN, int F>
__global__ void __launch_bounds__(THREADS, 1)
conv_stem_tc_fwd_kernel(const float* __restrict__ images, const float* __restrict__ kernel, const float* __restrict__ bias,
                        const pl::PlaneView pv, unsigned int* ovf,
                        uint32_t* __restrict__ argmax, int64_t B, int H, int W) {
  constexpr int K = 16 * CIN;              // 4x4xCIN patch
  constexpr int KB = (K + 31) / 32;        // k-blocks of 32 floats (128 B swizzle atoms)
  constexpr int N = 4 * F;                 // (pool position, filter)
  constexpr int NB = N * 128;              // bytes of one k-block of W'
  constexpr int NBUF = fwd_image_buffers(F);           // ring of staged images: the fetch of image i+NBUF-1 runs under image i
  constexpr int FJ = F / 8;                // 8-column fragment groups per pool position
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* s_w = base;                                  // [2 planes][KB][N][128 B]
  uint8_t* s_a = s_w + 2 * KB * NB;                     // [2 warpgroups][2 planes][KB][16 KB]
  const int pimg = (H + 2) * (W + 2) * CIN;
  float* s_img0 = reinterpret_cast<float*>(s_a + 2 * 2 * KB * TILE_BYTES);
  float* s_b = s_img0 + NBUF * pimg;

  const int tid = threadIdx.x, lane = tid & 31;
  const int slot = tid >> 7, r = tid & 127, wq = (tid >> 5) & 3;
  const int gid = lane >> 2, tq = lane & 3;
  // ---- once per CTA: W' (hi / lo, K-major swizzled), bias, zero borders of the image buffers ----
  for (int idx = tid; idx < N * K; idx += THREADS) {
    const int n = idx / K, k = idx - n * K;
    const int pos = n / F, f = n - pos * F;
    const int c = k % CIN, ij = k / CIN;
    const int ky = (ij >> 2) - (pos >> 1), kx = (ij & 3) - (pos & 1);
    const float v = (ky >= 0 && ky < 3 && kx >= 0 && kx < 3) ? kernel[((ky * 3 + kx) * CIN + c) * F + f] : 0.f;
    float h, l;
    pl::split_tf32(v, h, l);
    const uint32_t off = (uint32_t)(k >> 5) * NB + sw128(n, k & 31);
    *reinterpret_cast<float*>(s_w + off) = h;
    *reinterpret_cast<float*>(s_w + KB * NB + off) = l;
  }
  for (int i = tid; i < F; i += THREADS) s_b[i] = bias[i];
  for (int i = tid; i < NBUF * pimg; i += THREADS) s_img0[i] = 0.f;
  fence_async_smem();          // W' was written through the generic proxy, the MMAs read it through the async proxy
  __syncthreads();

  const int PH = H / 2, PW = W / 2, P = PH * PW;
  const int tiles = (P + 127) / 128;
  const int prow = (W + 2) * CIN;
  const int64_t img_elems = (int64_t)H * W * CIN;
  const int64_t words_per_row = (int64_t)P * F / 16;
  const uint32_t w_addr = smem_u32(s_w);
  uint8_t* a_hi = s_a + slot * (2 * KB * TILE_BYTES);
  uint8_t* a_lo = a_hi + KB * TILE_BYTES;
  const uint32_t a_addr = smem_u32(a_hi);
  int64_t b = blockIdx.x;
  for (int i = 0; i < NBUF - 1; ++i) {       // prologue: the first NBUF-1 images of this CTA
    const int64_t bi = b + (int64_t)i * gridDim.x;
    if (bi < B) stage_image<CIN>(s_img0 + i * pimg, images + bi * img_elems, H, W, tid);
    cp_async_commit();
  }
  int buf = 0;
  for (; b < B; b += gridDim.x, buf = (buf + 1 == NBUF) ? 0 : buf + 1) {
    cp_async_wait<NBUF - 2>();                       // this thread's copies of image b have landed
    __syncthreads();                                 // image b is visible to both warpgroups; image b-1 is no longer read
    const int64_t nb = b + (int64_t)(NBUF - 1) * gridDim.x;
    const int pbuf = (buf == 0) ? NBUF - 1 : buf - 1;    // the buffer image b-1 used
    if (nb < B) stage_image<CIN>(s_img0 + pbuf * pimg, images + nb * img_elems, H, W, tid);
    cp_async_commit();
    const float* s_img = s_img0 + buf * pimg;
    for (int tile = slot; tile < tiles; tile += 2) {
      {
        const int p = tile * 128 + r;
        const bool valid = p < P;
        const int py = valid ? p / PW : 0, px = valid ? p - py * PW : 0;
        const float* patch = s_img + (2 * py) * prow + (2 * px) * CIN;
        const uint32_t rowoff = (uint32_t)((r >> 3) * 1024 + (r & 7) * 128);
        wg_barrier(slot);                            // the previous tile's MMAs have finished reading this A buffer
#pragma unroll
        for (int q = 0; q < K / 4; ++q) {
          const int i = (CIN == 3) ? q / 3 : q;
          const int o = (CIN == 3) ? (q % 3) * 4 : 0;
          const float2 v0 = *reinterpret_cast<const float2*>(patch + i * prow + o);        // 8-byte aligned (W even)
          const float2 v1 = *reinterpret_cast<const float2*>(patch + i * prow + o + 2);
          float4 h4, l4;
          pl::split_tf32(v0.x, h4.x, l4.x);
          pl::split_tf32(v0.y, h4.y, l4.y);
          pl::split_tf32(v1.x, h4.z, l4.z);
          pl::split_tf32(v1.y, h4.w, l4.w);
          const uint32_t off = (uint32_t)(q >> 3) * TILE_BYTES + rowoff + (uint32_t)((((q & 7) ^ (r & 7)) & 7) << 4);
          *reinterpret_cast<float4*>(a_hi + off) = h4;
          *reinterpret_cast<float4*>(a_lo + off) = l4;
        }
        fence_async_smem();
        wg_barrier(slot);
      }
#pragma unroll 1
      for (int half = 0; half < 2; ++half) {
        float d[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
        wg::fence_regs(d);
        wg::fence();
#pragma unroll
        for (int prod = 0; prod < 3; ++prod) {       // a_hi b_hi, a_lo b_hi, a_hi b_lo
          const uint32_t aa = a_addr + (prod == 1 ? KB * TILE_BYTES : 0) + half * 8192;
          const uint32_t ww = w_addr + (prod == 2 ? KB * NB : 0);
#pragma unroll
          for (int ks = 0; ks < K / 8; ++ks)
            mma_tf32<N>(d, aa + (ks >> 2) * TILE_BYTES + (ks & 3) * 32, ww + (ks >> 2) * NB + (ks & 3) * 32,
                        (prod == 0 && ks == 0) ? 0u : 1u);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs(d);
        // ---- epilogue: rows 64 half + 16 wq + gid (+8); columns (pos, f) = 8 j + 2 tq + e, j = pos * FJ + fj ----
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int p = tile * 128 + 64 * half + 16 * wq + gid + 8 * rr;
          const bool valid = p < P;
#pragma unroll
          for (int g16 = 0; g16 < F / 16; ++g16) {
            uint32_t sign = 0u, arg = 0u;
#pragma unroll
            for (int h8 = 0; h8 < 2; ++h8) {
              const int fj = 2 * g16 + h8;
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int f = 8 * fj + 2 * tq + e;
                const float bv = s_b[f];
                float m = d[4 * fj + 2 * rr + e] + bv;
                uint32_t a = 0u;
#pragma unroll
                for (int pos = 1; pos < 4; ++pos) {
                  const float mp = d[4 * (pos * FJ + fj) + 2 * rr + e] + bv;
                  if (mp > m) { m = mp; a = (uint32_t)pos; }
                }
                m = fmaxf(m, 0.f);
                const int bit = f - 16 * g16;
                sign |= (m > 0.f) ? (1u << bit) : 0u;
                arg |= a << (2 * bit);
                if (valid) pl::plane_store(pv, b, p * F + f, m, ovf);
              }
            }
            sign |= __shfl_xor_sync(0xffffffffu, sign, 1);
            sign |= __shfl_xor_sync(0xffffffffu, sign, 2);
            arg |= __shfl_xor_sync(0xffffffffu, arg, 1);
            arg |= __shfl_xor_sync(0xffffffffu, arg, 2);
            if (valid && tq == 0) {
              const int64_t col0 = (int64_t)p * F + 16 * g16;
              reinterpret_cast<uint16_t*>(pv.bits)[((col0 >> 5) * B + b) * 2 + ((col0 >> 4) & 1)] = (uint16_t)sign;
              argmax[b * words_per_row + (col0 >> 4)] = arg;
            }
          }
        }
      }
    }
  }
}

template <int CIN, int F>
static size_t smem_bytes(int h, int w) {
  constexpr int K = 16 * CIN, KB = (K + 31) / 32, N = 4 * F;
  return 1024 + (size_t)2 * KB * N * 128 + (size_t)2 * 2 * KB * TILE_BYTES +
         (size_t)fwd_image_buffers(F) * (h + 2) * (w + 2) * CIN * 4 + F * 4;
}

template <int CIN, int F>
static int launch(const float* images, const float* kernel, const float* bias, const pl::PlaneView pv,
                  uint32_t* argmax, int64_t batch, int h, int w, cudaStream_t st) {
  const size_t smem = smem_bytes<CIN, F>(h, w);
  auto kern = conv_stem_tc_fwd_kernel<CIN, F>;
  const int64_t cap = sm_count();
  const int grid = (int)(batch < cap ? batch : cap);
  kern<<<grid, THREADS, smem, st>>>(images, kernel, bias, pv, pl::overflow_flag(), argmax, batch, h, w);
  ADN_CHECK_LAUNCH("conv_stem_tc_fwd");
  return ADN_OK;
}

// raised once from adn_init (never inside a stream capture, see conv::init)
int init() {
#define ADN_CONVTC_ATTR(K) ADN_CUDA(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024))
  ADN_CONVTC_ATTR((conv_stem_tc_fwd_kernel<1, 16>)); ADN_CONVTC_ATTR((conv_stem_tc_fwd_kernel<3, 16>));
  ADN_CONVTC_ATTR((conv_stem_tc_fwd_kernel<1, 32>)); ADN_CONVTC_ATTR((conv_stem_tc_fwd_kernel<3, 32>));
#undef ADN_CONVTC_ATTR
  return ADN_OK;
}

// true when the tensor-core path covers the shape (else the caller takes the SIMT kernel)
bool supported(int h, int w, int cin, int f) {
  if (f != 16 && f != 32) return false;
  const size_t smem = cin == 3 ? (f == 16 ? smem_bytes<3, 16>(h, w) : smem_bytes<3, 32>(h, w))
                               : (f == 16 ? smem_bytes<1, 16>(h, w) : smem_bytes<1, 32>(h, w));
  return smem <= 227 * 1024;
}

int fwd(const float* images, const float* kernel, const float* bias, void* out_planes, uint32_t* argmax, int64_t batch,
        int h, int w, int cin, int f, cudaStream_t st) {
  const int64_t cols = (int64_t)(h / 2) * (w / 2) * f;
  const pl::PlaneView pv = pl::plane_view(pl::format(), out_planes, batch, cols);
  if (cin == 3) return f == 16 ? launch<3, 16>(images, kernel, bias, pv, argmax, batch, h, w, st)
                               : launch<3, 32>(images, kernel, bias, pv, argmax, batch, h, w, st);
  return f == 16 ? launch<1, 16>(images, kernel, bias, pv, argmax, batch, h, w, st)
                 : launch<1, 32>(images, kernel, bias, pv, argmax, batch, h, w, st);
}

}  // namespace convtc
}  // namespace adn
