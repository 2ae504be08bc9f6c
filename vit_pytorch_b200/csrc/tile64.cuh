// The 64-row operand tile of the wgmma attention kernels that compute one 64 x 64 score block at a time
// (attention_tile64.cu, levit.cu, twins.cu's attention_kv, sep_vit.cu, regionvit.cu).  An operand block is 64 rows of one head's D columns:
// D / 64 slabs 64 columns wide with the 128B swizzle, then (D % 64) / 16 slabs 16 columns wide with the 32B swizzle.
// TMA boxes of 64 or 16 columns land in a slab as they are; cp.async gathers place 16-byte pieces at piece_addr.
// S = Q K^T reads Q and K blocks as K-major operands; O += P V takes P (bf16) from registers as the A operand and V as
// the transposed (MN-major) B operand, as in attention.cu.
#pragma once
#include "common.cuh"

namespace b200 {
namespace tile64 {

constexpr int ROWS = 64;
constexpr int THREADS = 128;  // one warpgroup

// One operand block of 64 rows: N64 slabs 64 columns wide (128B swizzle), then N16 slabs 16 columns wide (32B swizzle).
template <int D>
struct Slabs {
  static constexpr int N64 = D / 64;
  static constexpr int N16 = (D % 64) / 16;
  static_assert(N64 * 64 + N16 * 16 == D, "head width must be a multiple of 16");
  static constexpr int S64 = ROWS * 128;
  static constexpr int S16 = ROWS * 32;
  static constexpr int OP = N64 * S64 + N16 * S16;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// shared-memory address of the 16-byte piece c (columns 8c .. 8c + 7) of row r of an operand block at `base`
template <int D>
__device__ __forceinline__ uint32_t piece_addr(uint32_t base, int r, int c) {
  using S = Slabs<D>;
  if (c < S::N64 * 8) return base + (c >> 3) * S::S64 + r * 128 + (((c & 7) ^ (r & 7)) << 4);
  const int j = c - S::N64 * 8;
  return base + S::N64 * S::S64 + (j >> 1) * S::S16 + r * 32 + (((j & 1) ^ ((r >> 2) & 1)) << 4);
}

// rows r of an operand block from global rows src(r) (negative: zero-fill without a read), D columns from `col`;
// every thread of the warpgroup issues its share of cp.async pieces
template <int D, typename RowFn>
__device__ __forceinline__ void load_block(uint32_t base, const __nv_bfloat16* qkv, long long ld, int col, RowFn src,
                                           int tid) {
  constexpr int P = D / 8;
  for (int i = tid; i < ROWS * P; i += THREADS) {
    const int r = i / P, c = i - r * P;
    const long long row = src(r);
    const bool ok = row >= 0;
    cp_async16(piece_addr<D>(base, r, c), ok ? qkv + row * ld + col + 8 * c : qkv, ok);
  }
}

// S[64 x 64] = Q K^T over the slabs of one operand block each
template <int DK>
__device__ __forceinline__ void qk_mma(float (&s)[32], uint32_t sq, uint32_t sk) {
  using S = Slabs<DK>;
#pragma unroll
  for (int c = 0; c < S::N64; ++c)
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_m64n64k16(s, make_wgmma_desc(sq + c * S::S64, 1024, WGMMA_SW128) + 2 * k,
                      make_wgmma_desc(sk + c * S::S64, 1024, WGMMA_SW128) + 2 * k, c != 0 || k != 0);
#pragma unroll
  for (int c = 0; c < S::N16; ++c)
    wgmma_m64n64k16(s, make_wgmma_desc(sq + S::N64 * S::S64 + c * S::S16, 256, WGMMA_SW32),
                    make_wgmma_desc(sk + S::N64 * S::S64 + c * S::S16, 256, WGMMA_SW32), S::N64 != 0 || c != 0);
}

// O[64 x DV] += P V, P the 64 x 64 probabilities in this thread's S registers, V one operand block
template <int DV>
__device__ __forceinline__ void pv_mma(float (&o)[Slabs<DV>::N64 > 0 ? Slabs<DV>::N64 : 1][32],
                                       float (&o16)[Slabs<DV>::N16 > 0 ? Slabs<DV>::N16 : 1][8],
                                       const float (&s)[32], uint32_t sv) {
  using S = Slabs<DV>;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                           pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
#pragma unroll
    for (int c = 0; c < S::N64; ++c)
      wgmma_m64n64k16_rs_tb(o[c], a, make_wgmma_desc_lbo(sv + c * S::S64 + kk * 2048, 1024, 1024, WGMMA_SW128));
#pragma unroll
    for (int c = 0; c < S::N16; ++c)
      wgmma_m64n16k16_rs_tb(o16[c], a,
                            make_wgmma_desc_lbo(sv + S::N64 * S::S64 + c * S::S16 + kk * 512, 256, 256, WGMMA_SW32));
  }
}

// this thread's two row maxima, resp. row sums (rh), reduced over the four lanes that hold the row
__device__ __forceinline__ void quad_max(float (&mx)[2]) {
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 1));
    mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 2));
  }
}
__device__ __forceinline__ void quad_sum(float (&l)[2]) {
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 1);
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 2);
  }
}

// s <- exp2(s - mx) over a 64 x 64 score block in log2 units (s[4 jj + e]: row half e >> 1); l += this thread's part
// of each row's sum
__device__ __forceinline__ void tile_exp2(float (&s)[32], const float (&mx)[2], float (&l)[2]) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float v = fast_ex2(s[4 * jj + e] - mx[e >> 1]);
      s[4 * jj + e] = v;
      l[e >> 1] += v;
    }
}

// the plain softmax of a 64 x 64 score tile in place, keys c >= n dropped; l: this thread's two row sums
__device__ __forceinline__ void tile_softmax(float (&s)[32], float (&l)[2], int n, float scale_log2e, int lane) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = 8 * jj + 2 * (lane & 3) + (e & 1);
      s[4 * jj + e] = c < n ? s[4 * jj + e] * scale_log2e : -INFINITY;
      mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * jj + e]);
    }
  quad_max(mx);
  l[0] = l[1] = 0.f;
  tile_exp2(s, mx, l);
  quad_sum(l);
}

// O accumulators (pv_mma's) set to zero
template <int DH>
__device__ __forceinline__ void zero_acc(float (&o)[Slabs<DH>::N64 > 0 ? Slabs<DH>::N64 : 1][32],
                                         float (&o16)[Slabs<DH>::N16 > 0 ? Slabs<DH>::N16 : 1][8]) {
#pragma unroll
  for (int c = 0; c < Slabs<DH>::N64; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
#pragma unroll
  for (int c = 0; c < Slabs<DH>::N16; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) o16[c][i] = 0.f;
}

// this thread's two output rows (rh) of O, scaled by inv, to op (the row's first column of this head)
template <int DV>
__device__ __forceinline__ void store_rows(const float (&o)[Slabs<DV>::N64 > 0 ? Slabs<DV>::N64 : 1][32],
                                           const float (&o16)[Slabs<DV>::N16 > 0 ? Slabs<DV>::N16 : 1][8],
                                           __nv_bfloat16* op, int rh, float inv) {
  using S = Slabs<DV>;
#pragma unroll
  for (int c = 0; c < S::N64; ++c)
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
      *reinterpret_cast<uint32_t*>(op + 64 * c + jj * 8) =
          pack_bf16x2(o[c][4 * jj + 2 * rh] * inv, o[c][4 * jj + 2 * rh + 1] * inv);
#pragma unroll
  for (int c = 0; c < S::N16; ++c)
#pragma unroll
    for (int jj = 0; jj < 2; ++jj)
      *reinterpret_cast<uint32_t*>(op + 64 * S::N64 + 16 * c + jj * 8) =
          pack_bf16x2(o16[c][4 * jj + 2 * rh] * inv, o16[c][4 * jj + 2 * rh + 1] * inv);
}

}  // namespace tile64
}  // namespace b200
