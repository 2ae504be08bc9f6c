// The entry and the exit of the Compact Convolutional Transformer (reference cct.py) that no other kernel covers.
//
// b200vit_conv_im2col_nchw / _nhwc: the A operand of a zero-padded Conv2d(k, stride s, padding p) as a GEMM, written
//   with bit copies and zero fills (taps outside the image, and the K padding up to ldo, are zeros).  The first
//   tokenizer layer reads the NCHW image in column order (cin, ky, kx) -- F.unfold's order and the Conv2d weight's own
//   layout -- with one CTA per (image, output row, chunk of output columns) staging the input rows that output row
//   covers, zero halo included, in shared memory (the shape of unfold_kernel in pit.cu).  Later layers read the
//   channels-last bf16 output of the previous block in column order (ky, kx, cin), so every tap is a run of C
//   contiguous channels copied as 16-byte vectors, one warp per output row.
//
// b200vit_relu_maxpool: ReLU then MaxPool2d(pk, ps, pp) of the channels-last bf16 conv output as one pass,
//   relu(max(window)) (the two commute), padding counted as -inf and NaN propagated as F.max_pool2d does.  The result
//   is the bf16 channels-last input of the next conv layer, or the fp32 tokens [B*n, C] after the last one.
//
// b200vit_seq_pool: the final LayerNorm, attention_pool (Linear D -> 1), a softmax over each image's tokens and the
//   probability-weighted sum of the normalised tokens (cct.py:284-288), in fp32 with an online max.  A cluster of up
//   to 8 CTAs shares one image's rows; each warp keeps its own running (max, sum, accumulator), the CTA merges its
//   warps in shared memory and the cluster merges its CTAs through distributed shared memory, in a fixed order.
#include <cooperative_groups.h>

#include "common.cuh"
#include "host_util.h"

namespace cg = cooperative_groups;

namespace b200 {

// img [B, C, H, W] bf16; out row (b*oh + r)*ow + q, column (ch*k + i)*k + j = img[b, ch, r*s - p + i, q*s - p + j],
// or zero where that pixel is outside the image.  CTA (b*oh + r, chunk): output columns q0 .. q0 + nq - 1, which read
// image columns x0 = q0*s - p .. x0 + span - 1 of image rows r*s - p .. r*s - p + k - 1.
__global__ void __launch_bounds__(256)
im2col_nchw_kernel(const __nv_bfloat16* __restrict__ img, __nv_bfloat16* __restrict__ out, long long ldo, int C, int H,
                   int W, int k, int s, int p, int oh, int ow, int NQ, int CC) {
  extern __shared__ __nv_bfloat16 im2col_smem[];   // [cc][k][span], zero where the image has no pixel
  const int b = blockIdx.x / oh, r = blockIdx.x % oh;
  const int q0 = blockIdx.y * NQ;
  const int nq = ow - q0 < NQ ? ow - q0 : NQ;
  const int span = (nq - 1) * s + k, x0 = q0 * s - p, y0 = r * s - p, kk = k * k;
  const long long row0 = ((long long)b * oh + r) * ow + q0;
  const __nv_bfloat16* src = img + (long long)b * C * H * W;
  const __nv_bfloat16 zero = __float2bfloat16_rn(0.f);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  for (int c0 = 0; c0 < C; c0 += CC) {
    const int cc = C - c0 < CC ? C - c0 : CC;
    // one warp per staged row (c, i), its lanes along the row
    for (int ri = warp; ri < cc * k; ri += warps) {
      const int c = ri / k, i = ri - c * k, y = y0 + i;
      __nv_bfloat16* dst = im2col_smem + ri * span;
      if (y < 0 || y >= H) {
        for (int x = lane; x < span; x += 32) dst[x] = zero;
        continue;
      }
      const __nv_bfloat16* srow = src + (long long)(c0 + c) * H * W + (long long)y * W;
      for (int x = lane; x < span; x += 32) {
        const int xx = x0 + x;
        dst[x] = (xx >= 0 && xx < W) ? srow[xx] : zero;
      }
    }
    __syncthreads();
    // column t of the channel group comes from the same staged element for every output column of the chunk, shifted
    // by s per column: its position is worked out once and the chunk is walked
    const int seg = cc * kk;
    for (int t = threadIdx.x; t < seg; t += blockDim.x) {
      const int c = t / kk, rem = t - c * kk, i = rem / k, j = rem - i * k;
      const __nv_bfloat16* from = im2col_smem + (c * k + i) * span + j;
      __nv_bfloat16* to = out + row0 * ldo + (long long)c0 * kk + t;
      for (int q = 0; q < nq; ++q) to[q * ldo] = from[q * s];
    }
    __syncthreads();
  }
  const int K = C * kk, pad = (int)(ldo - K);
  for (int t = threadIdx.x; t < pad; t += blockDim.x)
    for (int q = 0; q < nq; ++q) out[(row0 + q) * ldo + K + t] = zero;
}

// x [B*H*W, C] bf16 channels-last (pixel (b, y, x) at row (b*H + y)*W + x), as CV = C / 8 16-byte vectors per row
// and LX8 16-byte vectors from one row to the next (LX8 >= CV: the rows may be a column slice of a wider buffer); out row (b*oh + r)*ow + q, vector (i*k + j)*CV + v = x[(b, r*s - p + i, q*s - p + j), vector v], or zeros outside
// the image; vectors [k*k*CV, ldo8) zero.  One warp per output row.
__global__ void __launch_bounds__(256)
im2col_nhwc_kernel(const uint4* __restrict__ x, long long lx8, uint4* __restrict__ out, long long ldo8, int H, int W,
                   int CV, int k, int s, int p, int oh, int ow, long long rows) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int q = (int)(row % ow);
  const long long t = row / ow;
  const int r = (int)(t % oh);
  const long long b = t / oh;
  const int y0 = r * s - p, x0 = q * s - p, kv = k * k * CV;
  const uint4* img = x + b * H * W * lx8;
  uint4* dst = out + row * ldo8;
  for (int v = lane; v < ldo8; v += 32) {
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (v < kv) {
      const int tap = v / CV, cv = v - tap * CV, i = tap / k, j = tap - i * k;
      const int y = y0 + i, xx = x0 + j;
      if (y >= 0 && y < H && xx >= 0 && xx < W) val = __ldg(img + ((long long)y * W + xx) * lx8 + cv);
    }
    dst[v] = val;
  }
}

// y [B*H*W, C] bf16 channels-last; out pixel (b, r, q) = relu(max of y over the pixels (r*ps - pp + i, q*ps - pp + j),
// i, j < pk, inside the image), channels-last, row stride ldo elements.  One thread per (output pixel, 8 channels).
template <bool F32>
__global__ void __launch_bounds__(256)
relu_maxpool_kernel(const uint4* __restrict__ y, void* __restrict__ out, long long ldo, int H, int W, int CV, int pk,
                    int ps, int pp, int oh, int ow, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = (int)(idx % CV);
  const long long row = idx / CV;
  const int q = (int)(row % ow);
  const long long t = row / ow;
  const int r = (int)(t % oh);
  const long long b = t / oh;
  const int ya = r * ps - pp, xa = q * ps - pp;
  const int y0 = ya > 0 ? ya : 0, y1 = ya + pk < H ? ya + pk : H;
  const int x0 = xa > 0 ? xa : 0, x1 = xa + pk < W ? xa + pk : W;
  float m[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) m[e] = -INFINITY;
  const uint4* img = y + b * H * W * CV + cv;
  for (int yy = y0; yy < y1; ++yy)
    for (int xx = x0; xx < x1; ++xx) {
      const uint4 v = __ldg(img + ((long long)yy * W + xx) * CV);
      const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        m[2 * e] = nan_max(m[2 * e], __uint_as_float(w4[e] << 16));
        m[2 * e + 1] = nan_max(m[2 * e + 1], __uint_as_float(w4[e] & 0xFFFF0000u));
      }
    }
#pragma unroll
  for (int e = 0; e < 8; ++e) m[e] = (m[e] > 0.f || m[e] != m[e]) ? m[e] : 0.f;   // ReLU, NaN kept
  if (F32) {
    float4* o = reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + row * ldo + cv * 8);
    o[0] = make_float4(m[0], m[1], m[2], m[3]);
    o[1] = make_float4(m[4], m[5], m[6], m[7]);
  } else {
    // the values are bf16 already: the packing is exact
    uint4 o;
    o.x = pack_bf16x2(m[0], m[1]);
    o.y = pack_bf16x2(m[2], m[3]);
    o.z = pack_bf16x2(m[4], m[5]);
    o.w = pack_bf16x2(m[6], m[7]);
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(out) + row * ldo + cv * 8) = o;
  }
}

// x fp32 [B*n, D], token t of image b at row b*n + t.  Cluster (of S CTAs) b: image b; CTA rank r takes tokens
// [r*per, (r + 1)*per), its warps every W-th of them.  Lane l owns channels 4l + 128j, j < J (D <= 128 J).
//   y_t = LN(x_t) (gamma g, beta be, eps),  z_t = y_t . wp + bp[0],  out[b] = sum_t softmax(z)_t y_t  (bf16)
template <int J>
__global__ void __launch_bounds__(256)
seq_pool_kernel(const float* __restrict__ x, int n, int D, const float* __restrict__ g, const float* __restrict__ be,
                float eps, const float* __restrict__ wp, const float* __restrict__ bp, __nv_bfloat16* __restrict__ out,
                long long ldo) {
  cg::cluster_group cluster = cg::this_cluster();
  const int S = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
  extern __shared__ float4 seq_pool_smem4[];
  float* acc_s = reinterpret_cast<float*>(seq_pool_smem4);   // [W][D]: each warp's accumulator, then the CTA's in row 0
  __shared__ float wm[8], wl[8];                               // each warp's running max and sum
  __shared__ float cta[2];                                    // the CTA's (max, sum), read by the whole cluster
  const int per = (n + S - 1) / S, t0 = rank * per, t1 = t0 + per < n ? t0 + per : n;
  const float bias = __ldg(bp);
  float4 acc[J];
#pragma unroll
  for (int j = 0; j < J; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  float m = -INFINITY, l = 0.f;
  for (int t = t0 + warp; t < t1; t += W) {
    const float* xr = x + ((long long)b * n + t) * D;
    float4 v[J];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int c = 4 * lane + 128 * j;
      v[j] = c < D ? *reinterpret_cast<const float4*>(xr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
    }
    const float mean = warp_sum(s) / (float)D;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      if (4 * lane + 128 * j < D) {
        const float a0 = v[j].x - mean, a1 = v[j].y - mean, a2 = v[j].z - mean, a3 = v[j].w - mean;
        q += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
      }
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)D + eps);
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int c = 4 * lane + 128 * j;
      if (c < D) {
        const float4 gg = __ldg(reinterpret_cast<const float4*>(g + c));
        const float4 bb = __ldg(reinterpret_cast<const float4*>(be + c));
        const float4 ww = __ldg(reinterpret_cast<const float4*>(wp + c));
        v[j].x = fmaf((v[j].x - mean) * rstd, gg.x, bb.x);
        v[j].y = fmaf((v[j].y - mean) * rstd, gg.y, bb.y);
        v[j].z = fmaf((v[j].z - mean) * rstd, gg.z, bb.z);
        v[j].w = fmaf((v[j].w - mean) * rstd, gg.w, bb.w);
        dot = fmaf(v[j].x, ww.x, fmaf(v[j].y, ww.y, fmaf(v[j].z, ww.z, fmaf(v[j].w, ww.w, dot))));
      }
    }
    const float z = warp_sum(dot) + bias;
    const float mn = nan_max(m, z);
    const float sc = l == 0.f ? 0.f : expf(m - mn), e = expf(z - mn);
#pragma unroll
    for (int j = 0; j < J; ++j) {
      acc[j].x = fmaf(acc[j].x, sc, e * v[j].x);
      acc[j].y = fmaf(acc[j].y, sc, e * v[j].y);
      acc[j].z = fmaf(acc[j].z, sc, e * v[j].z);
      acc[j].w = fmaf(acc[j].w, sc, e * v[j].w);
    }
    l = fmaf(l, sc, e);
    m = mn;
  }
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int c = 4 * lane + 128 * j;
    if (c < D) *reinterpret_cast<float4*>(acc_s + warp * D + c) = acc[j];
  }
  if (lane == 0) {
    wm[warp] = m;
    wl[warp] = l;
  }
  __syncthreads();
  // the CTA's warps, in warp order.  l == 0: a warp without tokens, which contributes nothing (its max is -inf).  A
  // NaN in any token of the image makes its max, and so every weight, NaN.
  float M = -INFINITY;
  for (int w = 0; w < W; ++w)
    if (wl[w] != 0.f) M = nan_max(M, wm[w]);
  float L = 0.f;
  for (int w = 0; w < W; ++w)
    if (wl[w] != 0.f) L = fmaf(wl[w], expf(wm[w] - M), L);
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float a = 0.f;
    for (int w = 0; w < W; ++w)
      if (wl[w] != 0.f) a = fmaf(acc_s[w * D + c], expf(wm[w] - M), a);
    acc_s[c] = a;
  }
  if (threadIdx.x == 0) {
    cta[0] = M;
    cta[1] = L;
  }
  cluster.sync();
  // the cluster's CTAs, in rank order; CTA `rank` writes channels rank*blockDim + tid, stride S*blockDim
  float Mg = -INFINITY;
  for (int q = 0; q < S; ++q) {
    const float* o = cluster.map_shared_rank(cta, q);
    if (o[1] != 0.f) Mg = nan_max(Mg, o[0]);
  }
  float Lg = 0.f;
  for (int q = 0; q < S; ++q) {
    const float* o = cluster.map_shared_rank(cta, q);
    if (o[1] != 0.f) Lg = fmaf(o[1], expf(o[0] - Mg), Lg);
  }
  for (int c = rank * blockDim.x + threadIdx.x; c < D; c += S * blockDim.x) {
    float a = 0.f;
    for (int q = 0; q < S; ++q) {
      const float* o = cluster.map_shared_rank(cta, q);
      if (o[1] != 0.f) a = fmaf(cluster.map_shared_rank(acc_s, q)[c], expf(o[0] - Mg), a);
    }
    out[(long long)b * ldo + c] = __float2bfloat16_rn(a / Lg);
  }
  cluster.sync();   // every CTA's shared memory stays until the whole cluster has read it
}

template <int J>
static cudaError_t launch_seq_pool(int S, int B, size_t smem, cudaStream_t st, const float* x, int n, int D,
                                   const float* g, const float* be, float eps, const float* wp, const float* bp,
                                   void* out, long long ldo) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)S, (unsigned)B);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)S;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, seq_pool_kernel<J>, x, n, D, g, be, eps, wp, bp,
                            reinterpret_cast<__nv_bfloat16*>(out), ldo);
}

}  // namespace b200

using namespace b200;

static constexpr int kIm2colSmem = 48 * 1024;

static bool al16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

extern "C" int b200vit_conv_im2col_nchw(const void* img, void* out_bf16, int64_t ldo, int B, int C, int H, int W,
                                        int k, int s, int p, void* stream) {
  B200_CHECK_ARG(img && out_bf16, "conv_im2col_nchw: null pointer");
  B200_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && k >= 1 && k <= B200VIT_CONV_MAX_KERNEL && s >= 1 && p >= 0 &&
                     p < k && H + 2 * p >= k && W + 2 * p >= k,
                 "conv_im2col_nchw: bad shape B=%d C=%d H=%d W=%d k=%d s=%d p=%d (1 <= k <= %d, s >= 1, 0 <= p < k, "
                 "H + 2p and W + 2p >= k)", B, C, H, W, k, s, p, B200VIT_CONV_MAX_KERNEL);
  const int oh = (H + 2 * p - k) / s + 1, ow = (W + 2 * p - k) / s + 1;
  const long long K = (long long)C * k * k, rows = (long long)B * oh * ow;
  B200_CHECK_ARG(ldo >= K && (ldo & 7) == 0, "conv_im2col_nchw: ldo=%lld must be a multiple of 8 and >= C*k*k=%lld",
                 (long long)ldo, K);
  B200_CHECK_ARG(rows * ldo <= (1LL << 40) && (long long)B * oh <= 0x7fffffff && (long long)B * C * H * W <= (1LL << 40),
                 "conv_im2col_nchw: %lld output pixels too many", rows);
  B200_CHECK_ARG(al16(out_bf16) && (reinterpret_cast<uintptr_t>(img) & 1) == 0,
                 "conv_im2col_nchw: out_bf16 must be 16-byte aligned, img 2-byte aligned");
  // all channels at once if one output pixel of them fits, else as many channels as fit; then as many output columns
  const long long per_c = (long long)k * sizeof(__nv_bfloat16);
  int cc = C;
  if (cc * per_c * k > kIm2colSmem) cc = (int)(kIm2colSmem / (per_c * k));
  const long long max_span = kIm2colSmem / (per_c * cc);
  int nq = (int)((max_span - k) / s + 1);
  if (nq > ow) nq = ow;
  const size_t smem = (size_t)cc * k * ((nq - 1) * s + k) * sizeof(__nv_bfloat16);
  const dim3 grid((unsigned)(B * oh), (unsigned)((ow + nq - 1) / nq));
  B200_CHECK_ARG(grid.y <= 65535, "conv_im2col_nchw: %d output columns too many", ow);
  im2col_nchw_kernel<<<grid, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(img), reinterpret_cast<__nv_bfloat16*>(out_bf16), (long long)ldo, C, H, W,
      k, s, p, oh, ow, nq, cc);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_conv_im2col_nhwc_ex(const void* x, int64_t ldx, int64_t M, void* out_bf16, int64_t ldo, int B,
                                           int H, int W, int C, int k, int s, int p, void* stream) {
  B200_CHECK_ARG(x && out_bf16, "conv_im2col_nhwc: null pointer");
  B200_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && k >= 1 && k <= B200VIT_CONV_MAX_KERNEL && s >= 1 && p >= 0 &&
                     p < k && H + 2 * p >= k && W + 2 * p >= k,
                 "conv_im2col_nhwc: bad shape B=%d H=%d W=%d C=%d k=%d s=%d p=%d (1 <= k <= %d, s >= 1, 0 <= p < k, "
                 "H + 2p and W + 2p >= k)", B, H, W, C, k, s, p, B200VIT_CONV_MAX_KERNEL);
  B200_CHECK_ARG(C % 8 == 0, "conv_im2col_nhwc: C=%d must be a multiple of 8", C);
  B200_CHECK_ARG(ldx >= C && (ldx & 7) == 0, "conv_im2col_nhwc: ldx=%lld must be a multiple of 8 and >= C=%d",
                 (long long)ldx, C);
  B200_CHECK_ARG(M == (long long)B * H * W, "conv_im2col_nhwc: x has %lld rows, B*H*W = %lld expected", (long long)M,
                 (long long)B * H * W);
  const int oh = (H + 2 * p - k) / s + 1, ow = (W + 2 * p - k) / s + 1;
  const long long K = (long long)C * k * k, rows = (long long)B * oh * ow;
  B200_CHECK_ARG(ldo >= K && (ldo & 7) == 0, "conv_im2col_nhwc: ldo=%lld must be a multiple of 8 and >= k*k*C=%lld",
                 (long long)ldo, K);
  B200_CHECK_ARG(rows * ldo <= (1LL << 40) && M * ldx <= (1LL << 40), "conv_im2col_nhwc: %lld output pixels too many",
                 rows);
  B200_CHECK_ARG(al16(x) && al16(out_bf16), "conv_im2col_nhwc: x and out_bf16 must be 16-byte aligned");
  const long long grid = (rows + 7) / 8;
  B200_CHECK_ARG(grid <= 0x7fffffff, "conv_im2col_nhwc: %lld CTAs too many", grid);
  im2col_nhwc_kernel<<<(unsigned)grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint4*>(x), (long long)ldx / 8, reinterpret_cast<uint4*>(out_bf16), (long long)ldo / 8, H,
      W, C / 8, k, s, p, oh, ow, rows);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_conv_im2col_nhwc(const void* x, int64_t M, void* out_bf16, int64_t ldo, int B, int H, int W,
                                        int C, int k, int s, int p, void* stream) {
  return b200vit_conv_im2col_nhwc_ex(x, C, M, out_bf16, ldo, B, H, W, C, k, s, p, stream);
}

extern "C" int b200vit_relu_maxpool(const void* y, int64_t M, int B, int H, int W, int C, int pk, int ps, int pp,
                                    void* out_bf16, float* out_f32, int64_t ldo, void* stream) {
  B200_CHECK_ARG(y && ((out_bf16 != nullptr) != (out_f32 != nullptr)),
                 "relu_maxpool: null pointer (y and exactly one of out_bf16 / out_f32)");
  B200_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && pk >= 1 && pk <= B200VIT_POOL_MAX_KERNEL && ps >= 1 && pp >= 0 &&
                     pp <= pk / 2 && H + 2 * pp >= pk && W + 2 * pp >= pk,
                 "relu_maxpool: bad shape B=%d H=%d W=%d C=%d pk=%d ps=%d pp=%d (1 <= pk <= %d, ps >= 1, "
                 "0 <= pp <= pk/2, H + 2pp and W + 2pp >= pk)", B, H, W, C, pk, ps, pp, B200VIT_POOL_MAX_KERNEL);
  B200_CHECK_ARG(C % 8 == 0, "relu_maxpool: C=%d must be a multiple of 8", C);
  B200_CHECK_ARG(M == (long long)B * H * W, "relu_maxpool: y has %lld rows, B*H*W = %lld expected", (long long)M,
                 (long long)B * H * W);
  B200_CHECK_ARG(ldo >= C && (ldo & (out_f32 ? 3 : 7)) == 0,
                 "relu_maxpool: ldo=%lld must be >= C=%d and a multiple of %d", (long long)ldo, C, out_f32 ? 4 : 8);
  B200_CHECK_ARG(al16(y) && al16(out_bf16) && al16(out_f32), "relu_maxpool: y and the output must be 16-byte aligned");
  const int oh = (H + 2 * pp - pk) / ps + 1, ow = (W + 2 * pp - pk) / ps + 1;
  const long long total = (long long)B * oh * ow * (C / 8);
  B200_CHECK_ARG(M * C <= (1LL << 40) && (total + 255) / 256 <= 0x7fffffff, "relu_maxpool: %lld pixels too many",
                 (long long)M);
  const unsigned grid = (unsigned)((total + 255) / 256);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  if (out_f32)
    relu_maxpool_kernel<true><<<grid, 256, 0, st>>>(reinterpret_cast<const uint4*>(y), out_f32, (long long)ldo, H, W,
                                                    C / 8, pk, ps, pp, oh, ow, total);
  else
    relu_maxpool_kernel<false><<<grid, 256, 0, st>>>(reinterpret_cast<const uint4*>(y), out_bf16, (long long)ldo, H, W,
                                                     C / 8, pk, ps, pp, oh, ow, total);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_seq_pool(const float* x, int B, int n, int D, const float* gamma, const float* beta, float eps,
                                const float* w, const float* bias, void* out_bf16, int64_t ldo, void* stream) {
  B200_CHECK_ARG(x && gamma && beta && w && bias && out_bf16, "seq_pool: null pointer");
  B200_CHECK_ARG(B > 0 && n > 0 && D > 0, "seq_pool: bad shape B=%d n=%d D=%d", B, n, D);
  B200_CHECK_ARG(D % 8 == 0 && D <= B200VIT_SEQ_POOL_MAX_DIM, "seq_pool: D=%d must be a multiple of 8 and <= %d", D,
                 B200VIT_SEQ_POOL_MAX_DIM);
  B200_CHECK_ARG(B <= 65535 && (long long)B * n * D <= (1LL << 40), "seq_pool: B=%d images of %d tokens too many", B, n);
  B200_CHECK_ARG(ldo >= D && (ldo & 7) == 0, "seq_pool: ldo=%lld must be a multiple of 8 and >= D=%d", (long long)ldo,
                 D);
  B200_CHECK_ARG(al16(x) && al16(gamma) && al16(beta) && al16(w) && al16(out_bf16),
                 "seq_pool: x, gamma, beta, w and out_bf16 must be 16-byte aligned");
  // as many CTAs per image (up to a cluster of 8) as fill about two waves, each warp still taking 8 tokens or more
  const int sms = num_sms();
  int S = (2 * sms + B - 1) / B;
  const int by_rows = n / (8 * 8);
  if (S > by_rows) S = by_rows;
  if (S > 8) S = 8;
  if (S < 1) S = 1;
  const size_t smem = (size_t)8 * D * sizeof(float);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  cudaError_t e;
  if (D <= 128) e = launch_seq_pool<1>(S, B, smem, st, x, n, D, gamma, beta, eps, w, bias, out_bf16, ldo);
  else if (D <= 512) e = launch_seq_pool<4>(S, B, smem, st, x, n, D, gamma, beta, eps, w, bias, out_bf16, ldo);
  else e = launch_seq_pool<8>(S, B, smem, st, x, n, D, gamma, beta, eps, w, bias, out_bf16, ldo);
  B200_CHECK_CUDA(e);
  count_launch();
  return 0;
}
