// The level boundaries of NesT (reference nest.py), for sm_90a.  Inside a level the fp32 residual stream is kept in
// the reference's own token order, block-major: a level whose H x W map is cut into nb x nb blocks of sh x sw tokens
// (sh = H/nb, sw = W/nb) holds token (b, y, x) at row
//   ((b*nb + y/sh)*nb + x/sw)*(sh*sw) + (y % sh)*sw + (x % sw)
// ('b c (b1 h) (b2 w) -> (b b1 b2) c h w', then the '(x y)' flattening inside Attention), so every level's encoder
// layers are a plain encoder over B*nb*nb sequences of sh*sw tokens.  The two kernels here are the only places the
// layout is read or written across blocks.
//
// b200vit_nest_level_entry: the start of every level.  The fp32 output of a GEMM in map order (the patch embedding's
//   1 x 1 convolution, or Aggregate's 3 x 3 convolution) -> LayerNorm over the channels of every pixel -> MaxPool2d
//   (pk, ps, pp) over the normalised values -> + pos_emb[r] (r the token's place inside its block) -> the next level's
//   stream in block-major order, and in LN-fold mode its bf16 copy and row statistics through emit_row_stats
//   (common.cuh), the bits b200vit_rowstats_cast would write.  The order is the reference's: LN, then the pool
//   (nest.py:76-81), then the position (nest.py:97-99).  One warp per output pixel: the LayerNorm statistics of the
//   pk*pk window pixels first, then per group of channels the max over the window of the normalised values.  The
//   pool counts padding as -inf and keeps a NaN once it has seen one, as F.max_pool2d does.
//
// b200vit_nest_im2col: the A operand of Aggregate's Conv2d(dim, dim_out, 3, padding = 1) as a GEMM, read from the
//   block-major stream and written in map order: row (b*H + y)*W + x, column (i*3 + j)*D + c (the order of
//   b200vit_conv_im2col_nhwc) the bf16 rounding of channel c of pixel (y - 1 + i, x - 1 + j), zero outside the map and
//   in the K padding.  One warp per output row, 8 channels per lane and step.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

// the row of token (b, y, x) in the block-major stream of nb x nb blocks of sh x sw tokens
__device__ __forceinline__ long long block_major_row(long long b, int y, int x, int nb, int sh, int sw) {
  return ((b * nb + y / sh) * nb + x / sw) * (long long)(sh * sw) + (y % sh) * sw + (x % sw);
}

// y fp32 [B*H*W, D] map order; output pixel (b, r, q) of the oh x ow pooled map to its block-major row of x (and xb,
// stats).  PK: the pool's kernel size, so the window's statistics stay in registers.
template <int PK>
__global__ void __launch_bounds__(256)
nest_level_entry_kernel(const float* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                        float eps, const float* __restrict__ pos, float* __restrict__ x, __nv_bfloat16* __restrict__ xb,
                        float* __restrict__ stats, int D, int H, int W, int ps, int pp, int oh, int ow, int nb,
                        long long rows) {
  constexpr int T = PK * PK;
  const long long pix = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (pix >= rows) return;
  const int lane = threadIdx.x & 31;
  const int q = (int)(pix % ow);
  const long long t = pix / ow;
  const int r = (int)(t % oh);
  const long long b = t / oh;
  const int ya = r * ps - pp, xa = q * ps - pp;
  const int y0 = ya > 0 ? ya : 0, y1 = ya + PK < H ? ya + PK : H;
  const int x0 = xa > 0 ? xa : 0, x1 = xa + PK < W ? xa + PK : W;
  const int nx = x1 - x0, nt = (y1 - y0) * nx;
  const float* img = y + b * H * W * D;
  const float* tap[T];
  float mean[T], rstd[T];
#pragma unroll
  for (int k = 0; k < T; ++k) {
    tap[k] = img;
    mean[k] = rstd[k] = 0.f;
    if (k < nt) {
      tap[k] = img + ((long long)(y0 + k / nx) * W + x0 + k % nx) * D;
      ln_row_stats(tap[k], D, lane, mean[k], rstd[k], eps);
    }
  }
  const int sh = oh / nb, sw = ow / nb;
  const long long orow = block_major_row(b, r, q, nb, sh, sw);
  const float pv = __ldg(pos + (r % sh) * sw + (q % sw));
  emit_row_stats<true>(
      D, lane, x + orow * D, xb ? xb + orow * D : nullptr, stats ? stats + 2 * orow : nullptr,
      [&](int i) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + i));
        const float4 be = __ldg(reinterpret_cast<const float4*>(beta + i));
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
        for (int k = 0; k < T; ++k) {
          if (k < nt) {
            const float4 v = *reinterpret_cast<const float4*>(tap[k] + i);
            m.x = nan_max(m.x, (v.x - mean[k]) * rstd[k] * g.x + be.x);
            m.y = nan_max(m.y, (v.y - mean[k]) * rstd[k] * g.y + be.y);
            m.z = nan_max(m.z, (v.z - mean[k]) * rstd[k] * g.z + be.z);
            m.w = nan_max(m.w, (v.w - mean[k]) * rstd[k] * g.w + be.w);
          }
        }
        return make_float4(m.x + pv, m.y + pv, m.z + pv, m.w + pv);
      },
      [&](int i) {
        const float g = __ldg(gamma + i), be = __ldg(beta + i);
        float m = -INFINITY;
#pragma unroll
        for (int k = 0; k < T; ++k)
          if (k < nt) m = nan_max(m, (tap[k][i] - mean[k]) * rstd[k] * g + be);
        return m + pv;
      });
}

// x fp32 [B*H*W, D] block-major as float4s (CV = D / 8 pairs of them per row); out [B*H*W, ldo8 16-byte vectors] bf16
// in map order, vector (i*3 + j)*CV + v = channels 8v .. 8v + 7 of pixel (y - 1 + i, x - 1 + j), zeros outside the map
// and from 9*CV on.
__global__ void __launch_bounds__(256)
nest_im2col_kernel(const float4* __restrict__ x, uint4* __restrict__ out, long long ldo8, int H, int W, int CV, int nb,
                   long long rows) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int px = (int)(row % W);
  const long long t = row / W;
  const int py = (int)(t % H);
  const long long b = t / H;
  const int sh = H / nb, sw = W / nb, kv = 9 * CV;
  uint4* dst = out + row * ldo8;
  for (int v = lane; v < ldo8; v += 32) {
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (v < kv) {
      const int tap = v / CV, cv = v - tap * CV, i = tap / 3, j = tap - 3 * i;
      const int yy = py - 1 + i, xx = px - 1 + j;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
        const float4* src = x + block_major_row(b, yy, xx, nb, sh, sw) * (2 * CV) + 2 * cv;
        const float4 a = __ldg(src), c = __ldg(src + 1);
        val = make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(c.x, c.y), pack_bf16x2(c.z, c.w));
      }
    }
    dst[v] = val;
  }
}

}  // namespace b200

using namespace b200;

static bool al16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

static bool overlap(const void* a, long long a_bytes, const void* b, long long b_bytes) {
  const uintptr_t p = reinterpret_cast<uintptr_t>(a), q = reinterpret_cast<uintptr_t>(b);
  return p < q + (uintptr_t)b_bytes && q < p + (uintptr_t)a_bytes;
}

extern "C" int b200vit_nest_level_entry(const float* y, int64_t M, const float* gamma, const float* beta, float eps,
                                        const float* pos, int n_pos, float* x, void* xb_bf16, float* stats, int B,
                                        int H, int W, int D, int pk, int ps, int pp, int nb, void* stream) {
  B200_CHECK_ARG(y && gamma && beta && pos && x, "nest_level_entry: null pointer");
  B200_CHECK_ARG((xb_bf16 != nullptr) == (stats != nullptr),
                 "nest_level_entry: the bf16 copy and the row statistics go together (both or neither)");
  B200_CHECK_ARG(B > 0 && H > 0 && W > 0 && D > 0 && pk >= 1 && pk <= B200VIT_NEST_POOL_MAX_KERNEL && ps >= 1 &&
                     pp >= 0 && pp <= pk / 2 && H + 2 * pp >= pk && W + 2 * pp >= pk,
                 "nest_level_entry: bad shape B=%d H=%d W=%d D=%d pk=%d ps=%d pp=%d (1 <= pk <= %d, ps >= 1, "
                 "0 <= pp <= pk/2, H + 2pp and W + 2pp >= pk)", B, H, W, D, pk, ps, pp, B200VIT_NEST_POOL_MAX_KERNEL);
  B200_CHECK_ARG(M == (long long)B * H * W, "nest_level_entry: y has %lld rows, B*H*W = %lld expected", (long long)M,
                 (long long)B * H * W);
  const int oh = (H + 2 * pp - pk) / ps + 1, ow = (W + 2 * pp - pk) / ps + 1;
  B200_CHECK_ARG(nb >= 1 && oh % nb == 0 && ow % nb == 0,
                 "nest_level_entry: the %d x %d pooled map does not split into %d x %d blocks", oh, ow, nb, nb);
  const int n_block = (oh / nb) * (ow / nb);
  B200_CHECK_ARG(n_pos >= n_block, "nest_level_entry: %d positions for blocks of %d tokens", n_pos, n_block);
  const long long rows = (long long)B * oh * ow;
  B200_CHECK_ARG(M * D <= (1LL << 40) && (rows + 7) / 8 <= 0x7fffffff, "nest_level_entry: %lld pixels too many",
                 (long long)M);
  B200_CHECK_ARG(al16(y) && al16(x) && al16(xb_bf16) && al16(gamma) && al16(beta),
                 "nest_level_entry: y, x, the bf16 copy, gamma and beta must be 16-byte aligned");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(stats) & 7) == 0, "nest_level_entry: stats must be 8-byte aligned");
  B200_CHECK_ARG(!overlap(y, M * D * 4, x, rows * D * 4) &&
                     !(xb_bf16 && overlap(y, M * D * 4, xb_bf16, rows * D * 2)),
                 "nest_level_entry: the outputs overlap y");
  const unsigned grid = (unsigned)((rows + 7) / 8);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  auto xb = reinterpret_cast<__nv_bfloat16*>(xb_bf16);
  if (pk == 1)
    nest_level_entry_kernel<1><<<grid, 256, 0, st>>>(y, gamma, beta, eps, pos, x, xb, stats, D, H, W, ps, pp, oh, ow,
                                                     nb, rows);
  else if (pk == 2)
    nest_level_entry_kernel<2><<<grid, 256, 0, st>>>(y, gamma, beta, eps, pos, x, xb, stats, D, H, W, ps, pp, oh, ow,
                                                     nb, rows);
  else
    nest_level_entry_kernel<3><<<grid, 256, 0, st>>>(y, gamma, beta, eps, pos, x, xb, stats, D, H, W, ps, pp, oh, ow,
                                                     nb, rows);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_nest_im2col(const float* x, int64_t M, void* out_bf16, int64_t ldo, int B, int H, int W, int D,
                                   int nb, void* stream) {
  B200_CHECK_ARG(x && out_bf16, "nest_im2col: null pointer");
  B200_CHECK_ARG(B > 0 && H > 0 && W > 0 && D > 0 && D % 8 == 0,
                 "nest_im2col: bad shape B=%d H=%d W=%d D=%d (D a multiple of 8)", B, H, W, D);
  B200_CHECK_ARG(M == (long long)B * H * W, "nest_im2col: x has %lld rows, B*H*W = %lld expected", (long long)M,
                 (long long)B * H * W);
  B200_CHECK_ARG(nb >= 1 && H % nb == 0 && W % nb == 0,
                 "nest_im2col: the %d x %d map does not split into %d x %d blocks", H, W, nb, nb);
  B200_CHECK_ARG(ldo >= 9LL * D && (ldo & 7) == 0, "nest_im2col: ldo=%lld must be a multiple of 8 and >= 9*D=%lld",
                 (long long)ldo, 9LL * D);
  B200_CHECK_ARG(M * ldo <= (1LL << 40) && (M + 7) / 8 <= 0x7fffffff, "nest_im2col: %lld pixels too many",
                 (long long)M);
  B200_CHECK_ARG(al16(x) && al16(out_bf16), "nest_im2col: x and out_bf16 must be 16-byte aligned");
  B200_CHECK_ARG(!overlap(x, M * D * 4, out_bf16, M * ldo * 2), "nest_im2col: out_bf16 overlaps x");
  nest_im2col_kernel<<<(unsigned)((M + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<uint4*>(out_bf16), (long long)ldo / 8, H, W, D / 8, nb, M);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
