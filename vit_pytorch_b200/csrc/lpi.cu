// Local patch interaction (XCiT's LPI, reference xcit.py:150-167) on the h x w token grid of every image, out of place:
//   y = x + conv2'(GELU(conv1'(LN(x))))
// conv1' and conv2' are depthwise k x k convolutions with zero padding k / 2.  The host folds BatchNorm (eval) into
// conv1' and LayerScale into conv2'; the LayerNorm's gamma / beta stay separate because the padding pads the
// LayerNorm OUTPUT (a border tap sees 0, not beta).  Likewise conv2's padding pads the GELU output: intermediate values
// outside the grid are set to 0, never evaluated.
//
// Two launches:
//   lpi_ln_stats_kernel: one warp per token, (mean, 1 / sqrt(var + eps)) of x into a [M][2] scratch;
//   lpi_kernel<K, CH>:   one CTA per (image, band of up to 4 grid rows r0 .. r1).  Channel chunk by channel chunk (CH
//                        channels), it stages z = LN(x) for grid rows r0 - 2p .. r1 + 2p and columns -p .. w - 1 + p in
//                        shared memory (zeros outside the grid), computes u = GELU(conv1'(z)) for rows r0 - p .. r1 + p
//                        (zeros outside the grid), then y = x + conv2'(u) for the tokens of rows r0 .. r1.  After
//                        the last chunk every warp turns finished rows of y into their bf16 copy and row statistics with rowstats_cast_row, the
//                        device code of b200vit_rowstats_cast, so the LN-folded fc1 GEMM reads the same bits it would
//                        read after that kernel.
// Each output token reads its neighbours' input rows, so y must not overlap x.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

__global__ void __launch_bounds__(256)
lpi_ln_stats_kernel(const float* __restrict__ x, float* __restrict__ ms, int M, int D, float eps) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  float mean, rstd;
  ln_row_stats(x + row * D, D, lane, mean, rstd, eps);
  if (lane == 0) {
    ms[2 * row] = mean;
    ms[2 * row + 1] = rstd;
  }
}

__device__ __forceinline__ float gelu_exact(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f)); }

// w1, w2: fp32 [K*K][D] (tap-major, so consecutive threads read consecutive channels); b1, b2: fp32 [D].
// Thread t owns channel c0 + t % CH of every chunk (its 2 K^2 weights live in registers) and walks the positions
// t / CH, t / CH + 256 / CH, ... of a row.  One CTA covers RB grid rows, so the z and u halos are shared by them.
template <int K, int CH>
__global__ void __launch_bounds__(256)
lpi_kernel(const float* __restrict__ x, const float* __restrict__ ms, const float* __restrict__ gamma,
           const float* __restrict__ beta, const float* __restrict__ w1, const float* __restrict__ b1,
           const float* __restrict__ w2, const float* __restrict__ b2, float* __restrict__ y,
           __nv_bfloat16* __restrict__ yb, float* __restrict__ ystats, int gh, int gw, int D, int RB) {
  constexpr int P = K / 2;
  constexpr int PL = 256 / CH;    // position lanes
  const int WP = gw + 2 * P;      // padded row: columns -P .. gw - 1 + P
  const int bands = (gh + RB - 1) / RB;
  const int b = blockIdx.x / bands, r0 = (blockIdx.x % bands) * RB;
  const int rb = gh - r0 < RB ? gh - r0 : RB;      // grid rows of this CTA
  extern __shared__ float4 lpi_smem4[];
  float* zs = reinterpret_cast<float*>(lpi_smem4);   // [rb + 4P][WP][CH]  z rows r0 - 2P ..
  float* us = zs + (RB + 4 * P) * WP * CH;           // [rb + 2P][WP][CH]  u rows r0 - P ..
  const int tid = threadIdx.x, ch = tid % CH, pl = tid / CH;
  const long long img0 = (long long)b * gh * gw;     // first token of the image
  for (int c0 = 0; c0 < D; c0 += CH) {
    const int c = c0 + ch;
    float w1r[K * K], w2r[K * K];
#pragma unroll
    for (int i = 0; i < K * K; ++i) {
      w1r[i] = w1[i * D + c];
      w2r[i] = w2[i * D + c];
    }
    const float g = gamma[c], bt = beta[c], bias1 = b1[c], bias2 = b2[c];
    for (int zr = 0; zr < rb + 4 * P; ++zr) {
      const int rr = r0 - 2 * P + zr;
      for (int pc = pl; pc < WP; pc += PL) {
        const int col = pc - P;
        float v = 0.f;
        if (rr >= 0 && rr < gh && col >= 0 && col < gw) {
          const long long tok = img0 + (long long)rr * gw + col;
          v = fmaf((x[tok * D + c] - ms[2 * tok]) * ms[2 * tok + 1], g, bt);
        }
        zs[(zr * WP + pc) * CH + ch] = v;
      }
    }
    __syncthreads();
    for (int ur = 0; ur < rb + 2 * P; ++ur) {
      const int rr = r0 - P + ur;
      for (int pc = pl; pc < WP; pc += PL) {
        const int col = pc - P;
        float v = 0.f;
        if (rr >= 0 && rr < gh && col >= 0 && col < gw) {
          float acc = bias1;
#pragma unroll
          for (int dy = 0; dy < K; ++dy)
#pragma unroll
            for (int dx = 0; dx < K; ++dx)
              acc = fmaf(w1r[dy * K + dx], zs[((ur + dy) * WP + col + dx) * CH + ch], acc);
          v = gelu_exact(acc);
        }
        us[(ur * WP + pc) * CH + ch] = v;
      }
    }
    __syncthreads();
    for (int orow = 0; orow < rb; ++orow) {
      for (int col = pl; col < gw; col += PL) {
        float acc = bias2;
#pragma unroll
        for (int dy = 0; dy < K; ++dy)
#pragma unroll
          for (int dx = 0; dx < K; ++dx)
            acc = fmaf(w2r[dy * K + dx], us[((orow + dy) * WP + col + dx) * CH + ch], acc);
        const long long o = (img0 + (long long)(r0 + orow) * gw + col) * D + c;
        y[o] = x[o] + acc;
      }
    }
    __syncthreads();
  }
  if (yb != nullptr) {
    const int warp = tid >> 5, lane = tid & 31;
    for (int i = warp; i < rb * gw; i += 8) {
      const long long tok = img0 + (long long)r0 * gw + i;
      rowstats_cast_row(y + tok * D, yb + tok * D, ystats + 2 * tok, D, lane);
    }
  }
}

// grid rows per CTA and the widest channel chunk that divides D and keeps the z and u slabs within 100 KB of shared
// memory (chunk 0: none fits, even one row per CTA)
static int lpi_tiling(int k, int gh, int gw, int D, int* rows, size_t* smem) {
  const int p = k / 2;
  for (int rb = gh < 4 ? gh : 4;; rb = 1) {
    for (int ch = 32; ch >= 4; ch /= 2) {
      const size_t s = (size_t)(2 * rb + 6 * p) * (size_t)(gw + 2 * p) * ch * sizeof(float);
      if (D % ch == 0 && s <= 100 * 1024) {
        *rows = rb;
        *smem = s;
        return ch;
      }
    }
    if (rb == 1) return 0;
  }
}

template <int K, int CH>
static int launch_lpi_kernel(int grid, size_t smem, cudaStream_t st, const float* x, const float* ms,
                             const float* gamma, const float* beta, const float* w1, const float* b1, const float* w2,
                             const float* b2, float* y, void* yb, float* ystats, int gh, int gw, int D, int rb) {
  const auto kern = lpi_kernel<K, CH>;
  B200_ENSURE_SMEM(kern, smem);
  kern<<<grid, 256, smem, st>>>(x, ms, gamma, beta, w1, b1, w2, b2, y, reinterpret_cast<__nv_bfloat16*>(yb), ystats,
                                gh, gw, D, rb);
  return 0;
}

template <int K>
static int launch_lpi(int ch, int grid, size_t smem, cudaStream_t st, const float* x, const float* ms,
                      const float* gamma, const float* beta, const float* w1, const float* b1, const float* w2,
                      const float* b2, float* y, void* yb, float* ystats, int gh, int gw, int D, int rb) {
  switch (ch) {
    case 32:
      return launch_lpi_kernel<K, 32>(grid, smem, st, x, ms, gamma, beta, w1, b1, w2, b2, y, yb, ystats, gh, gw, D, rb);
    case 16:
      return launch_lpi_kernel<K, 16>(grid, smem, st, x, ms, gamma, beta, w1, b1, w2, b2, y, yb, ystats, gh, gw, D, rb);
    case 8:
      return launch_lpi_kernel<K, 8>(grid, smem, st, x, ms, gamma, beta, w1, b1, w2, b2, y, yb, ystats, gh, gw, D, rb);
    default:
      return launch_lpi_kernel<K, 4>(grid, smem, st, x, ms, gamma, beta, w1, b1, w2, b2, y, yb, ystats, gh, gw, D, rb);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200vit_local_patch_interaction(const float* x, float* y, void* y_bf16, float* y_stats,
                                               float* ln_scratch, const float* ln_gamma, const float* ln_beta,
                                               float ln_eps, const float* w1, const float* b1, const float* w2,
                                               const float* b2, int B, int gh, int gw, int D, int k, void* stream) {
  B200_CHECK_ARG(x && y && ln_scratch && ln_gamma && ln_beta && w1 && b1 && w2 && b2,
                 "local_patch_interaction: null pointer");
  B200_CHECK_ARG((y_bf16 == nullptr) == (y_stats == nullptr),
                 "local_patch_interaction: y_bf16 and y_stats are both given or both null");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && D > 0, "local_patch_interaction: bad shape B=%d h=%d w=%d D=%d", B, gh,
                 gw, D);
  B200_CHECK_ARG(k == 1 || k == 3 || k == 5 || k == 7,
                 "local_patch_interaction: kernel size %d not supported by this build (1, 3, 5 or 7)", k);
  B200_CHECK_ARG(D % 4 == 0, "local_patch_interaction: D=%d must be a multiple of 4", D);
  const long long M = (long long)B * gh * gw;
  B200_CHECK_ARG(M <= 0x7fffffff && M * D <= (1LL << 40) && (long long)B * gh <= 0x7fffffff,
                 "local_patch_interaction: %lld tokens too many", M);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(y_bf16) & 7) == 0,
                 "local_patch_interaction: x and y must be 16-byte aligned, y_bf16 8-byte aligned");
  const auto xa = reinterpret_cast<uintptr_t>(x), ya = reinterpret_cast<uintptr_t>(y);
  const uintptr_t bytes = (uintptr_t)(M * D) * sizeof(float);
  B200_CHECK_ARG(ya + bytes <= xa || xa + bytes <= ya,
                 "local_patch_interaction: y overlaps x (every token reads its neighbours' rows of x)");
  size_t smem = 0;
  int rb = 1;
  const int ch = lpi_tiling(k, gh, gw, D, &rb, &smem);
  B200_CHECK_ARG(ch > 0, "local_patch_interaction: a grid row of %d tokens does not fit in shared memory", gw);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  lpi_ln_stats_kernel<<<(int)((M + 7) / 8), 256, 0, st>>>(x, ln_scratch, (int)M, D, ln_eps);
  B200_CHECK_CUDA(cudaGetLastError());
  const int grid = B * ((gh + rb - 1) / rb);
  int rc;
  switch (k) {
    case 1: rc = launch_lpi<1>(ch, grid, smem, st, x, ln_scratch, ln_gamma, ln_beta, w1, b1, w2, b2, y, y_bf16,
                               y_stats, gh, gw, D, rb); break;
    case 3: rc = launch_lpi<3>(ch, grid, smem, st, x, ln_scratch, ln_gamma, ln_beta, w1, b1, w2, b2, y, y_bf16,
                               y_stats, gh, gw, D, rb); break;
    case 5: rc = launch_lpi<5>(ch, grid, smem, st, x, ln_scratch, ln_gamma, ln_beta, w1, b1, w2, b2, y, y_bf16,
                               y_stats, gh, gw, D, rb); break;
    default: rc = launch_lpi<7>(ch, grid, smem, st, x, ln_scratch, ln_gamma, ln_beta, w1, b1, w2, b2, y, y_bf16,
                                y_stats, gh, gw, D, rb);
  }
  if (rc) return rc;
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return 0;
}
