// Kernels of CrossFormer (reference crossformer.py), for sm_90a.
//   b200vit_cross_embed_nchw   the stage-1 cross-scale embedding (CrossEmbedLayer, crossformer.py:14-36): up to four
//                              convolutions of the NCHW image with different kernel sizes and one stride, their
//                              channels concatenated, written as the fp32 channels-last stream
//
// An implicit GEMM on wgmma.  One CTA = two warpgroups = an 8 x 16 block of output tokens of one image (warpgroup g
// takes its rows 4g .. 4g + 3: one 64-row M tile).  The CTA stages the input band those tokens cover, halo included and
// zero outside the image, in shared memory once.  Then, scale after scale and k-block after k-block (64 columns of the
// scale's K = C*k*k, in the order (channel, tap row, tap column) of Conv2d's weight), every thread gathers its token's
// 32 columns from the band into the warpgroup's A tile and the CTA copies the scale's packed weight rows into the B
// tile, both 128B-swizzled and double buffered: the gather of k-block t + 1 runs under the MMAs of k-block t.  Each
// scale's accumulators (m64n8k16 per 8 output channels, fp32) start from zero, and after its last k-block the bias is
// added and the tokens' columns [off, off + n) are stored.  No im2col matrix is written, sums run in a fixed order and
// nothing is atomic.
#include "common.cuh"
#include "host_util.h"

namespace {

using namespace b200;

constexpr int CE_THREADS = 256;
constexpr int CE_TR = 8, CE_TC = 16;         // output tokens of a CTA: 8 rows x 16 columns
constexpr int CE_TILE_BYTES = 64 * 128;      // 64 rows x 64 bf16, 128B swizzle (A per warpgroup, B per CTA)
constexpr int CE_STAGE_BYTES = 3 * CE_TILE_BYTES;
constexpr int CE_BAND_OFF = 2 * CE_STAGE_BYTES;

struct CrossEmbedParams {
  const uint16_t* img;
  const __nv_bfloat16* w;
  const float* bias;
  float* out;
  long long ldo;
  int C, H, W, oh, ow, s, S, pmax, rows, cols, tiles_x, tiles;
  int k[B200VIT_CROSS_EMBED_MAX_SCALES], n[B200VIT_CROSS_EMBED_MAX_SCALES], off[B200VIT_CROSS_EMBED_MAX_SCALES];
  long long woff[B200VIT_CROSS_EMBED_MAX_SCALES];
};

// D[64 x 8] (+)= A[64 x 16] * B[8 x 16]^T, both K-major in shared memory (see wgmma_m64n128k16)
__device__ __forceinline__ void wgmma_m64n8k16(float (&d)[4], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %6, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

__device__ __forceinline__ uint32_t swz(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

__global__ void __launch_bounds__(CE_THREADS)
cross_embed_kernel(const CrossEmbedParams p) {
  extern __shared__ __align__(1024) uint8_t ce_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ce_smem_raw) + 1023) & ~uintptr_t(1023));
  uint16_t* band = reinterpret_cast<uint16_t*>(smem + CE_BAND_OFF);

  const int tid = threadIdx.x;
  const int b = blockIdx.x / p.tiles, tile = blockIdx.x % p.tiles;
  const int r0 = (tile / p.tiles_x) * CE_TR, q0 = (tile % p.tiles_x) * CE_TC;

  // the input band of the CTA's tokens: rows r0*s - pmax + [0, rows), columns q0*s - pmax + [0, cols), per channel
  {
    const int gy0 = r0 * p.s - p.pmax, gx0 = q0 * p.s - p.pmax;
    const int per_c = p.rows * p.cols, total = p.C * per_c;
    const uint16_t* src = p.img + (size_t)b * p.C * p.H * p.W;
    for (int e = tid; e < total; e += CE_THREADS) {
      const int c = e / per_c, rem = e - c * per_c;
      const int y = rem / p.cols, x = rem - y * p.cols;
      const int gy = gy0 + y, gx = gx0 + x;
      uint16_t v = 0;
      if (gy >= 0 && gy < p.H && gx >= 0 && gx < p.W) v = __ldg(src + ((size_t)c * p.H + gy) * p.W + gx);
      band[e] = v;
    }
  }
  __syncthreads();

  const int wg = tid >> 7, lt = tid & 127;
  // A gather: token m of the warpgroup's tile, k columns half*32 .. half*32 + 31 of every k-block
  const int m = lt & 63, half = lt >> 6;
  const int tr = wg * 4 + (m >> 4), tc = m & 15;
  const bool valid = r0 + tr < p.oh && q0 + tc < p.ow;

  float acc[8][4] = {};
  int it = 0;
  for (int sc = 0; sc < p.S; ++sc) {
    const int ks = p.k[sc], kk2 = ks * ks, Ks = p.C * kk2, ng = p.n[sc] >> 3;
    const int kp16 = (Ks + 15) & ~15, kp = (Ks + 63) & ~63, nkb = kp >> 6;
    const int d = p.pmax - (ks - p.s) / 2;                 // this scale's window origin inside the band
    const uint16_t* tb = band + (tr * p.s + d) * p.cols + tc * p.s + d;
    const __nv_bfloat16* wsrc = p.w + p.woff[sc];
    for (int kb = 0; kb < nkb; ++kb, ++it) {
      uint8_t* stage = smem + (it & 1) * CE_STAGE_BYTES;
      uint8_t* A = stage + wg * CE_TILE_BYTES;
      uint8_t* Bt = stage + 2 * CE_TILE_BYTES;
      {
        int k = kb * 64 + half * 32;
        int c = k / kk2, rem = k - c * kk2;
        int i = rem / ks, j = rem - i * ks;
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
          uint32_t pk[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            uint32_t lo = 0, hi = 0;
            if (valid && k < Ks) lo = tb[(c * p.rows + i) * p.cols + j];
            ++k;
            if (++j == ks) { j = 0; if (++i == ks) { i = 0; ++c; } }
            if (valid && k < Ks) hi = tb[(c * p.rows + i) * p.cols + j];
            ++k;
            if (++j == ks) { j = 0; if (++i == ks) { i = 0; ++c; } }
            pk[e] = lo | (hi << 16);
          }
          sts_v4(smem_u32(A) + swz(m, half * 4 + ch), pk[0], pk[1], pk[2], pk[3]);
        }
      }
      for (int e = tid; e < ng * 64; e += CE_THREADS) {
        const int row = e >> 3, ch = e & 7;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(wsrc + (size_t)row * kp + kb * 64 + ch * 8));
        sts_v4(smem_u32(Bt) + swz(row, ch), v.x, v.y, v.z, v.w);
      }
      fence_proxy_async_smem();
      __syncthreads();

      const int steps = min(4, (kp16 - kb * 64) >> 4);
      wgmma_fence();
#pragma unroll
      for (int s16 = 0; s16 < 4; ++s16) {
        if (s16 < steps) {
          const uint64_t da = make_wgmma_desc(smem_u32(A) + s16 * 32, 1024, WGMMA_SW128);
          const uint32_t first = (kb > 0 || s16 > 0) ? 1u : 0u;
#pragma unroll
          for (int g = 0; g < 8; ++g)
            if (g < ng)
              wgmma_m64n8k16(acc[g], da, make_wgmma_desc(smem_u32(Bt) + g * 1024 + s16 * 32, 1024, WGMMA_SW128),
                             first);
        }
      }
      wgmma_commit();
      if (kb + 1 < nkb) {
        wgmma_wait<1>();
      } else {
        wgmma_wait<0>();
#pragma unroll
        for (int g = 0; g < 8; ++g) fence_regs(acc[g]);
        // epilogue: rows lane/4 and lane/4 + 8 of the warp's 16, columns 2*(lane%4) + {0, 1} of every 8
        const int warp = lt >> 5, lane = lt & 31;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int mm = warp * 16 + (lane >> 2) + hr * 8;
          const int rr = r0 + wg * 4 + (mm >> 4), qq = q0 + (mm & 15);
          if (rr < p.oh && qq < p.ow) {
            float* orow = p.out + ((long long)b * p.oh + rr) * p.ow * p.ldo + (long long)qq * p.ldo;
#pragma unroll
            for (int g = 0; g < 8; ++g) {
              if (g < ng) {
                const int col = p.off[sc] + g * 8 + 2 * (lane & 3);
                const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                *reinterpret_cast<float2*>(orow + col) = make_float2(acc[g][2 * hr] + bb.x, acc[g][2 * hr + 1] + bb.y);
              }
            }
          }
        }
      }
      // both warpgroups' MMAs on the other stage are done before anyone gathers into it
      __syncthreads();
    }
  }
}

}  // namespace

extern "C" int b200vit_cross_embed_nchw(const void* img, const void* w, const float* bias, float* out, int64_t ldo,
                                        int B, int C, int H, int W, int S, const int* ks, const int* ns, int s,
                                        void* stream) {
  B200_CHECK_ARG(img && w && bias && out && ks && ns, "cross_embed_nchw: null pointer");
  B200_CHECK_ARG(B > 0 && C >= 1 && C <= B200VIT_CROSS_EMBED_MAX_CHANNELS && H > 0 && W > 0,
                 "cross_embed_nchw: bad shape B=%d C=%d H=%d W=%d (C at most %d)", B, C, H, W,
                 B200VIT_CROSS_EMBED_MAX_CHANNELS);
  B200_CHECK_ARG(S >= 1 && S <= B200VIT_CROSS_EMBED_MAX_SCALES, "cross_embed_nchw: %d scales (1 to %d)", S,
                 B200VIT_CROSS_EMBED_MAX_SCALES);
  B200_CHECK_ARG(s >= 1 && s <= B200VIT_CROSS_EMBED_MAX_STRIDE, "cross_embed_nchw: stride %d (1 to %d)", s,
                 B200VIT_CROSS_EMBED_MAX_STRIDE);
  CrossEmbedParams p{};
  p.img = reinterpret_cast<const uint16_t*>(img);
  p.w = reinterpret_cast<const __nv_bfloat16*>(w);
  p.bias = bias;
  p.out = out;
  p.ldo = ldo;
  p.C = C; p.H = H; p.W = W; p.s = s; p.S = S;
  int dim = 0, pmax = 0, ext = 0;
  long long woff = 0;
  for (int i = 0; i < S; ++i) {
    const int k = ks[i], n = ns[i];
    B200_CHECK_ARG(k >= s && k <= B200VIT_CROSS_EMBED_MAX_KERNEL,
                   "cross_embed_nchw: scale %d kernel %d (from the stride %d to %d)", i, k, s,
                   B200VIT_CROSS_EMBED_MAX_KERNEL);
    B200_CHECK_ARG(n >= 8 && n <= B200VIT_CROSS_EMBED_MAX_WIDTH && n % 8 == 0,
                   "cross_embed_nchw: scale %d width %d (a multiple of 8 up to %d)", i, n, B200VIT_CROSS_EMBED_MAX_WIDTH);
    const int pad = (k - s) / 2;
    B200_CHECK_ARG(H + 2 * pad >= k && W + 2 * pad >= k, "cross_embed_nchw: scale %d kernel %d exceeds %d x %d", i, k,
                   H, W);
    const int oh = (H + 2 * pad - k) / s + 1, ow = (W + 2 * pad - k) / s + 1;
    if (i == 0) {
      p.oh = oh;
      p.ow = ow;
    }
    B200_CHECK_ARG(oh == p.oh && ow == p.ow, "cross_embed_nchw: scale %d maps to %d x %d, scale 0 to %d x %d", i, oh,
                   ow, p.oh, p.ow);
    p.k[i] = k;
    p.n[i] = n;
    p.off[i] = dim;
    p.woff[i] = woff;
    dim += n;
    woff += (long long)n * ((C * k * k + 63) / 64 * 64);
    pmax = pad > pmax ? pad : pmax;
  }
  for (int i = 0; i < S; ++i) {
    const int e = pmax - (ks[i] - s) / 2 + ks[i];
    ext = e > ext ? e : ext;
  }
  B200_CHECK_ARG(ldo >= dim && ldo % 2 == 0, "cross_embed_nchw: ldo=%lld (even, at least the width %d)",
                 (long long)ldo, dim);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(w) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0 &&
                     (reinterpret_cast<uintptr_t>(bias) & 7) == 0,
                 "cross_embed_nchw: w must be 16-byte aligned, out and bias 8-byte aligned");
  p.pmax = pmax;
  p.rows = (CE_TR - 1) * s + ext;
  p.cols = (CE_TC - 1) * s + ext;
  p.tiles_x = (p.ow + CE_TC - 1) / CE_TC;
  p.tiles = ((p.oh + CE_TR - 1) / CE_TR) * p.tiles_x;
  const long long grid = (long long)B * p.tiles;
  B200_CHECK_ARG(grid <= 0x7fffffffLL, "cross_embed_nchw: %lld tiles exceed the grid", grid);
  const size_t smem = 1024 + CE_BAND_OFF + (size_t)C * p.rows * p.cols * 2;
  B200_ENSURE_SMEM(cross_embed_kernel, smem);
  cross_embed_kernel<<<(unsigned)grid, CE_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
