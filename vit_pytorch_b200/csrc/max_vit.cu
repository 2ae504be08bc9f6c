// Kernels of MaxViT (reference max_vit.py), for sm_90a.  The token map of a stage is kept channels-last: x[B*h*w, C],
// token (b, y, x) at row (b*h + y)*w + x, whether the attention groups it into blocks or into dilated grids.  The
// window attention with its relative-position bias, b200vit_attention_window_relpos, is in attention_tile64.cu.
//   b200vit_mbconv_dwconv             depthwise 3 x 3 convolution, BatchNorm folded, GELU, and the per-image channel
//                                     sums squeeze-excitation averages (max_vit.py:106-109)
//   b200vit_mbconv_dwconv_ex          the same with GELU or SiLU and the sums optional (MobileViT's MV2Block,
//                                     mobile_vit.py:108-127)
//   b200vit_se_pool / b200vit_se_scale  the squeeze-excitation mean and gate around its two GEMMs (max_vit.py:47-62)
//
// mbconv_dwconv: one thread = two adjacent channels of one image over a run of B200VIT_MBCONV_PART_ROWS output
// tokens; a warp reads 64 consecutive channels of a token per tap (128 B).  The thread sums its bf16-rounded outputs
// in token order and writes the sum to its own slot of `part`, which se_pool adds up in part order.
#include "common.cuh"
#include "host_util.h"

namespace {

using namespace b200;

// ------------------------------------------------------------------------------------------------ mbconv_dwconv
constexpr int DW_THREADS = 128;

// y sigmoid(y), sigmoid(y) = 1 / (1 + 2^(-y log2 e)): the GEMM epilogue's EPI_SILU, so both give the same bits
__device__ __forceinline__ float silu_fast(float y) {
  return y * fast_rcp(1.0f + fast_ex2(-1.4426950408889634f * y));
}

// ACT: B200VIT_EPI_GELU or B200VIT_EPI_SILU; part NULL: no channel sums
template <int ACT>
__global__ void __launch_bounds__(DW_THREADS)
mbconv_dwconv_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w9, const float* __restrict__ bias,
                     __nv_bfloat16* __restrict__ y, float* __restrict__ part, int h, int w, int oh, int ow, int C,
                     int s, int P) {
  const int c = (blockIdx.x * DW_THREADS + threadIdx.x) * 2;
  if (c >= C) return;
  const int pi = blockIdx.y, b = blockIdx.z;
  const int n = oh * ow;
  const int t0 = pi * B200VIT_MBCONV_PART_ROWS;
  const int t1 = min(t0 + B200VIT_MBCONV_PART_ROWS, n);
  float2 wt[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) wt[k] = *reinterpret_cast<const float2*>(w9 + (long long)k * C + c);
  const float2 bb = *reinterpret_cast<const float2*>(bias + c);
  const __nv_bfloat16* xb = x + (long long)b * h * w * C + c;
  __nv_bfloat16* yb = y + (long long)b * n * C + c;
  float sum0 = 0.f, sum1 = 0.f;
  for (int t = t0; t < t1; ++t) {
    const int oy = t / ow, ox = t - (t / ow) * ow;
    float a0 = bb.x, a1 = bb.y;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = oy * s - 1 + ky;
      if (iy < 0 || iy >= h) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = ox * s - 1 + kx;
        if (ix < 0 || ix >= w) continue;
        const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(xb + ((long long)iy * w + ix) * C));
        a0 = fmaf(wt[3 * ky + kx].x, v.x, a0);
        a1 = fmaf(wt[3 * ky + kx].y, v.y, a1);
      }
    }
    if (ACT == B200VIT_EPI_GELU) {
      gelu_erf2(a0, a1);
    } else {
      a0 = silu_fast(a0);
      a1 = silu_fast(a1);
    }
    const uint32_t pk = pack_bf16x2(a0, a1);
    *reinterpret_cast<uint32_t*>(yb + (long long)t * C) = pk;
    sum0 += __uint_as_float(pk << 16);
    sum1 += __uint_as_float(pk & 0xFFFF0000u);
  }
  if (part) *reinterpret_cast<float2*>(part + ((long long)b * P + pi) * C + c) = make_float2(sum0, sum1);
}

// ------------------------------------------------------------------------------------------------ se_pool / se_scale
__global__ void __launch_bounds__(256)
se_pool_kernel(const float* __restrict__ part, __nv_bfloat16* __restrict__ pooled, int P, int C, float inv_n) {
  const int c = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
  if (c >= C) return;
  const float* pp = part + (long long)b * P * C + c;
  float sum = 0.f;
  for (int i = 0; i < P; ++i) sum += pp[(long long)i * C];
  pooled[(long long)b * C + c] = __float2bfloat16_rn(sum * inv_n);
}

// one thread per 8 channels of one token
__global__ void __launch_bounds__(256)
se_scale_kernel(__nv_bfloat16* __restrict__ hbuf, const __nv_bfloat16* __restrict__ gate, long long total8, int n,
                int C) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= total8) return;
  const int C8 = C >> 3;
  const long long tok = i / C8;
  const int c = (int)(i - tok * C8) * 8;
  const long long b = tok / n;
  uint4* hp = reinterpret_cast<uint4*>(hbuf + tok * C + c);
  uint4 hv = *hp;
  const uint4 gv = *reinterpret_cast<const uint4*>(gate + b * C + c);
  uint32_t* hw = reinterpret_cast<uint32_t*>(&hv);
  const uint32_t* gw = reinterpret_cast<const uint32_t*>(&gv);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hw[k]));
    const float2 gf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&gw[k]));
    hw[k] = pack_bf16x2(hf.x * gf.x, hf.y * gf.y);
  }
  *hp = hv;
}

}  // namespace

static inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

extern "C" int b200vit_mbconv_dwconv_ex(const void* x, int64_t M, const float* w9, const float* bias, void* y,
                                        float* part, int B, int h, int w, int C, int stride, int act, void* stream) {
  B200_CHECK_ARG(x && w9 && bias && y, "mbconv_dwconv: null pointer");
  B200_CHECK_ARG(act == B200VIT_EPI_GELU || act == B200VIT_EPI_SILU,
                 "mbconv_dwconv: act=%d (B200VIT_EPI_GELU or B200VIT_EPI_SILU)", act);
  B200_CHECK_ARG(B > 0 && h > 0 && w > 0 && C > 0, "mbconv_dwconv: bad shape B=%d h=%d w=%d C=%d", B, h, w, C);
  B200_CHECK_ARG(stride == 1 || stride == 2, "mbconv_dwconv: stride=%d (1 or 2)", stride);
  B200_CHECK_ARG(M == (int64_t)B * h * w, "mbconv_dwconv: x has %lld rows, %lld expected", (long long)M,
                 (long long)B * h * w);
  B200_CHECK_ARG(C % 8 == 0, "mbconv_dwconv: C=%d must be a multiple of 8", C);
  B200_CHECK_ARG(x != y, "mbconv_dwconv: y must not be x (every token reads its neighbours)");
  B200_CHECK_ARG(aligned16(x) && aligned16(w9) && aligned16(bias) && aligned16(y) && aligned16(part),
                 "mbconv_dwconv: pointers must be 16-byte aligned");
  const int oh = (h + stride - 1) / stride, ow = (w + stride - 1) / stride;
  const long long P = ((long long)oh * ow + B200VIT_MBCONV_PART_ROWS - 1) / B200VIT_MBCONV_PART_ROWS;
  B200_CHECK_ARG(B <= 65535 && P <= 65535, "mbconv_dwconv: B=%d, %lld parts exceed the grid", B, P);
  const dim3 grid((C / 2 + DW_THREADS - 1) / DW_THREADS, (unsigned)P, B);
  auto kern = act == B200VIT_EPI_GELU ? mbconv_dwconv_kernel<B200VIT_EPI_GELU> : mbconv_dwconv_kernel<B200VIT_EPI_SILU>;
  kern<<<grid, DW_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), w9, bias, reinterpret_cast<__nv_bfloat16*>(y), part, h, w, oh, ow, C,
      stride, (int)P);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_mbconv_dwconv(const void* x, int64_t M, const float* w9, const float* bias, void* y, float* part,
                                     int B, int h, int w, int C, int stride, void* stream) {
  B200_CHECK_ARG(part, "mbconv_dwconv: null pointer");
  return b200vit_mbconv_dwconv_ex(x, M, w9, bias, y, part, B, h, w, C, stride, B200VIT_EPI_GELU, stream);
}

extern "C" int b200vit_se_pool(const float* part, void* pooled, int B, int P, int C, float inv_n, void* stream) {
  B200_CHECK_ARG(part && pooled, "se_pool: null pointer");
  B200_CHECK_ARG(B > 0 && P > 0 && C > 0, "se_pool: bad shape B=%d P=%d C=%d", B, P, C);
  B200_CHECK_ARG(C % 8 == 0, "se_pool: C=%d must be a multiple of 8", C);
  B200_CHECK_ARG(aligned16(part) && aligned16(pooled), "se_pool: pointers must be 16-byte aligned");
  B200_CHECK_ARG(B <= 65535, "se_pool: B=%d exceeds the grid", B);
  se_pool_kernel<<<dim3((C + 255) / 256, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      part, reinterpret_cast<__nv_bfloat16*>(pooled), P, C, inv_n);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_se_scale(void* h, const void* gate, int B, int n, int C, void* stream) {
  B200_CHECK_ARG(h && gate, "se_scale: null pointer");
  B200_CHECK_ARG(B > 0 && n > 0 && C > 0, "se_scale: bad shape B=%d n=%d C=%d", B, n, C);
  B200_CHECK_ARG(C % 8 == 0, "se_scale: C=%d must be a multiple of 8", C);
  B200_CHECK_ARG(aligned16(h) && aligned16(gate), "se_scale: pointers must be 16-byte aligned");
  const long long total8 = (long long)B * n * (C / 8);
  B200_CHECK_ARG((total8 + 255) / 256 <= 0x7fffffffLL, "se_scale: %lld elements exceed the grid", total8 * 8);
  se_scale_kernel<<<(unsigned)((total8 + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<__nv_bfloat16*>(h), reinterpret_cast<const __nv_bfloat16*>(gate), total8, n, C);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
