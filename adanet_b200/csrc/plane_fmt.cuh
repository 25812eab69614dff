// Split-plane tensor formats of the tensor-core dense pipeline (planes.cu) and the helpers every kernel that
// WRITES planes shares (GEMM epilogues, head loss, optimizer, conv stem).
//
// A matrix T[rows, cols] (fp32) is held as two planes of 11-significant-bit values plus sign bits:
//
//   ADN_PLANES_F16  (default)  hi = fp16(T)        lo' = fp16((T - hi) * 2^11)       T ~= hi + 2^-11 lo'
//       2 B / value, k-block = 64 columns (one 128 B swizzle row), plane[cols/64][rows][64]
//       GEMMs issue fp16 wgmma (twice the tf32 rate):
//           H = sum a_hi b_hi,   S = sum (a_hi b_lo' + a_lo' b_hi),   C = H + 2^-11 S
//       fp16 carries 5 exponent bits: full 22-bit precision for 2^-14 <= |T| < 65504, absolute error 2^-36
//       below that; gradient tensors (O(1/batch)) are therefore carried multiplied by a power of two
//       (dz_log2_scale at the ABI) and un-scaled exactly where they leave the plane format (dW, db).
//       A finite |T| >= 65520 cannot be represented: the element-wise writers (input split, optimizer, head, conv
//       stem) raise the device-side sticky flag (adn_plane_overflow); a GEMM result beyond the range becomes Inf in
//       its output planes and surfaces as a non-finite loss.  Either way the host re-runs the iteration on TF32
//       planes (core/search.py restart_on_tf32_if_overflowed).
//   ADN_PLANES_TF32            hi = rna_tf32(T)    lo  = rna_tf32(T - hi)            T ~= hi + lo
//       4 B / value, k-block = 32 columns, plane[cols/32][rows][32]; tf32 MMAs; fp32 exponent range.
//
// Both: hi plane, lo plane, then sign bits  bits[ceil(cols/32)][rows]  (uint32, bit j = T[row, 32 q + j] > 0).
// The K padding (columns up to the k-block multiple) is zero.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace adn {
namespace pl {

enum { FMT_TF32 = ADN_PLANES_TF32, FMT_F16 = ADN_PLANES_F16 };

int format();                     // process-wide current format (adn_set_plane_format / ADN_PLANES)
unsigned int* overflow_flag();    // device address of the sticky overflow word (per process / device)

__host__ __device__ __forceinline__ int fmt_bk(int fmt) { return fmt == FMT_F16 ? 64 : 32; }
__host__ __device__ __forceinline__ int fmt_esize(int fmt) { return fmt == FMT_F16 ? 2 : 4; }

// elements in ONE plane (hi or lo) of a [rows, cols] tensor
inline int64_t plane_elems(int fmt, int64_t rows, int64_t cols) {
  return align_up(rows * ceil_div(cols, fmt_bk(fmt)) * fmt_bk(fmt), 128);
}
inline int64_t plane_bytes1(int fmt, int64_t rows, int64_t cols) { return plane_elems(fmt, rows, cols) * fmt_esize(fmt); }
// 32-column blocks the sign bits cover (whole k-blocks)
inline int64_t bits_blocks(int fmt, int64_t cols) { return ceil_div(cols, fmt_bk(fmt)) * (fmt_bk(fmt) / 32); }
inline int64_t bits_words(int fmt, int64_t rows, int64_t cols) { return align_up(rows * bits_blocks(fmt, cols), 64); }
inline int64_t planes_bytes(int fmt, int64_t rows, int64_t cols) {
  return 2 * plane_bytes1(fmt, rows, cols) + bits_words(fmt, rows, cols) * 4;
}

// Device-side view of a plane tensor for element-wise writers.
struct PlaneView {
  void* hi;
  void* lo;
  uint32_t* bits;
  int64_t rows;
  int fmt;
};
inline PlaneView plane_view(int fmt, void* planes, int64_t rows, int64_t cols) {
  char* p = reinterpret_cast<char*>(planes);
  const int64_t pb = plane_bytes1(fmt, rows, cols);
  return PlaneView{p, p + pb, reinterpret_cast<uint32_t*>(p + 2 * pb), rows, fmt};
}
inline const uint32_t* bits_of(int fmt, const void* planes, int64_t rows, int64_t cols) {
  return reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(planes) + 2 * plane_bytes1(fmt, rows, cols));
}

#ifdef __CUDACC__
// cvt.rna.tf32.f32 is emulated in SASS; on the bit pattern it is "add half a TF32 ulp to the magnitude, clear the low
// 13 bits".  Finite values round as cvt.rna does (FLT_MAX and its neighbours round to Inf) and Inf stays Inf, but a NaN
// whose top 11 mantissa bits are set carries through the exponent into the sign: the canonical NaN the GPU's own
// arithmetic produces, 0x7FFFFFFF, becomes -0.  Only split_tf32 below may see a NaN.
__device__ __forceinline__ float rna_tf32(float v) { return __uint_as_float((__float_as_uint(v) + 0x1000u) & 0xffffe000u); }
// hi = rna_tf32(v), lo = rna_tf32(v - hi) for finite v; a NaN keeps its bits in hi and +-Inf is hi = +-Inf, lo = 0, so
// that hi + lo is NaN / +-Inf again (rounding v - hi = NaN would make Inf's lo a NaN).
__device__ __forceinline__ void split_tf32(float v, float& hi, float& lo) {
  hi = rna_tf32(v);
  lo = rna_tf32(v - hi);
  if (!(fabsf(v) <= 3.402823466e38f)) {   // NaN or +-Inf: one compare with a free |.| modifier
    hi = v;
    lo = 0.f;
  }
}
// hi = fp16(v), lo' = fp16((v - hi) * 2^11): v - hi is exact in fp32 (hi is v rounded to 11 bits)
__device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
  hi = __float2half_rn(v);
  lo = __float2half_rn((v - __half2float(hi)) * 2048.0f);
}
__device__ __forceinline__ float merge_f16(__half hi, __half lo) { return fmaf(__half2float(lo), 1.0f / 2048.0f, __half2float(hi)); }
// finite but not representable in fp16 (rounds to Inf): 65520 <= |v| < Inf
__device__ __forceinline__ bool f16_overflows(float v) {
  const uint32_t m = __float_as_uint(v) & 0x7fffffffu;
  return m >= 0x477ff000u && m < 0x7f800000u;
}
__device__ __forceinline__ void raise_overflow(unsigned int* flag) { atomicOr(flag, 1u); }

// Element-wise store of T[r, c] = v into a plane tensor (both planes; sign bits are the caller's business).
__device__ __forceinline__ void plane_store(const PlaneView& p, int64_t r, int c, float v, unsigned int* ovf) {
  if (p.fmt == FMT_F16) {
    __half h, l;
    split_f16(v, h, l);
    if (f16_overflows(v)) raise_overflow(ovf);
    const int64_t dst = ((int64_t)(c >> 6) * p.rows + r) * 64 + (c & 63);
    reinterpret_cast<__half*>(p.hi)[dst] = h;
    reinterpret_cast<__half*>(p.lo)[dst] = l;
  } else {
    float h, l;
    split_tf32(v, h, l);
    const int64_t dst = ((int64_t)(c >> 5) * p.rows + r) * 32 + (c & 31);
    reinterpret_cast<float*>(p.hi)[dst] = h;
    reinterpret_cast<float*>(p.lo)[dst] = l;
  }
}
// T[r, c0 .. c0+7] = m[0..7] (c0 a multiple of 8): one 16 B (f16) or two 16 B (tf32) stores per plane
__device__ __forceinline__ void plane_store8(const PlaneView& p, int64_t r, int64_t c0, const float (&m)[8], unsigned int* ovf) {
  if (p.fmt == FMT_F16) {
    uint32_t hw[4], lw[4];
    bool over = false;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      __half h0, l0, h1, l1;
      split_f16(m[2 * q], h0, l0);
      split_f16(m[2 * q + 1], h1, l1);
      over |= f16_overflows(m[2 * q]) | f16_overflows(m[2 * q + 1]);
      hw[q] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
      lw[q] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
    }
    if (over) raise_overflow(ovf);
    const int64_t dst = ((c0 >> 6) * p.rows + r) * 64 + (c0 & 63);
    *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.hi) + dst) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.lo) + dst) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
  } else {
    float h[8], l[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) split_tf32(m[q], h[q], l[q]);
    const int64_t dst = ((c0 >> 5) * p.rows + r) * 32 + (c0 & 31);
    float* hp = reinterpret_cast<float*>(p.hi) + dst;
    float* lp = reinterpret_cast<float*>(p.lo) + dst;
    *reinterpret_cast<float4*>(hp) = make_float4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<float4*>(hp + 4) = make_float4(h[4], h[5], h[6], h[7]);
    *reinterpret_cast<float4*>(lp) = make_float4(l[0], l[1], l[2], l[3]);
    *reinterpret_cast<float4*>(lp + 4) = make_float4(l[4], l[5], l[6], l[7]);
  }
}
#endif

}  // namespace pl
}  // namespace adn
