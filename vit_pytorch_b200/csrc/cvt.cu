// Kernels of CvT (reference cvt.py), for sm_90a.  The token map of a stage is kept channels-last: x[B*h*w, C], token
// (b, y, x) at row (b*h + y)*w + x.
//   b200vit_conv_proj_dw   the depthwise halves of an attention layer's two convolutional projections (cvt.py:51-60,
//                          74-75): the k x k depthwise convolution + BatchNorm at stride 1 for the queries and at
//                          stride s for the keys / values, from one read of the LayerNorm'ed map
//
// Both convolutions have the same kernel size and padding k / 2, so key / value output (r, c) covers exactly the
// k x k neighbourhood of query output (s*r, s*c).  One thread = 8 channels (one 16-byte vector) of one query token: it
// gathers the neighbourhood once, always writes the query output and, on the stride lattice, also the key / value
// output from the same loaded values.  The weights (k*k*C fp32 per convolution) come out of L1 / L2.
#include "common.cuh"
#include "host_util.h"

namespace {

using namespace b200;

constexpr int CP_THREADS = 256;

__device__ __forceinline__ void load8(const float* __restrict__ p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ uint4 pack8(const float (&a)[8]) {
  uint4 r;
  r.x = pack_bf16x2(a[0], a[1]);
  r.y = pack_bf16x2(a[2], a[3]);
  r.z = pack_bf16x2(a[4], a[5]);
  r.w = pack_bf16x2(a[6], a[7]);
  return r;
}

template <int K>
__global__ void __launch_bounds__(CP_THREADS)
conv_proj_dw_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ wq, const float* __restrict__ bq,
                    const float* __restrict__ wkv, const float* __restrict__ bkv, __nv_bfloat16* __restrict__ q_out,
                    __nv_bfloat16* __restrict__ kv_out, long long total8, int h, int w, int oh, int ow, int C, int s) {
  const long long i = (long long)blockIdx.x * CP_THREADS + threadIdx.x;
  if (i >= total8) return;
  const int C8 = C >> 3;
  const int c = (int)(i % C8) * 8;
  const long long tok = i / C8;
  const int xx = (int)(tok % w);
  const long long by = tok / w;
  const int yy = (int)(by % h);
  const long long b = by / h;
  const bool lattice = (yy % s == 0) && (xx % s == 0);
  constexpr int R = K / 2;
  float aq[8], akv[8];
  load8(bq + c, aq);
  if (lattice) load8(bkv + c, akv);
#pragma unroll
  for (int dy = 0; dy < K; ++dy) {
    const int sy = yy + dy - R;
    if (sy < 0 || sy >= h) continue;
#pragma unroll
    for (int dx = 0; dx < K; ++dx) {
      const int sx = xx + dx - R;
      if (sx < 0 || sx >= w) continue;
      const uint4 raw = *reinterpret_cast<const uint4*>(x + (tok + (long long)(dy - R) * w + (dx - R)) * C + c);
      const uint32_t* rw = reinterpret_cast<const uint32_t*>(&raw);
      float v[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        v[2 * e] = __uint_as_float(rw[e] << 16);
        v[2 * e + 1] = __uint_as_float(rw[e] & 0xFFFF0000u);
      }
      float wt[8];
      load8(wq + (long long)(dy * K + dx) * C + c, wt);
#pragma unroll
      for (int e = 0; e < 8; ++e) aq[e] = fmaf(wt[e], v[e], aq[e]);
      if (lattice) {
        load8(wkv + (long long)(dy * K + dx) * C + c, wt);
#pragma unroll
        for (int e = 0; e < 8; ++e) akv[e] = fmaf(wt[e], v[e], akv[e]);
      }
    }
  }
  *reinterpret_cast<uint4*>(q_out + tok * C + c) = pack8(aq);
  if (lattice) {
    const long long row = (b * oh + yy / s) * ow + xx / s;
    *reinterpret_cast<uint4*>(kv_out + row * C + c) = pack8(akv);
  }
}

}  // namespace

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static inline bool overlap(const void* a, long long na, const void* b, long long nb) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return pa < pb + (uintptr_t)nb && pb < pa + (uintptr_t)na;
}

extern "C" int b200vit_conv_proj_dw(const void* x, int64_t M, const float* wq, const float* bq, const float* wkv,
                                    const float* bkv, void* q_out, void* kv_out, int B, int h, int w, int C, int k,
                                    int s, void* stream) {
  B200_CHECK_ARG(x && wq && bq && wkv && bkv && q_out && kv_out, "conv_proj_dw: null pointer");
  B200_CHECK_ARG(B > 0 && h > 0 && w > 0 && C > 0, "conv_proj_dw: bad shape B=%d h=%d w=%d C=%d", B, h, w, C);
  B200_CHECK_ARG(k == 1 || k == 3 || k == 5 || k == 7, "conv_proj_dw: kernel size %d not built (1, 3, 5 or 7)", k);
  B200_CHECK_ARG(s >= 1, "conv_proj_dw: stride s=%d must be >= 1", s);
  B200_CHECK_ARG(C % 8 == 0, "conv_proj_dw: C=%d must be a multiple of 8", C);
  B200_CHECK_ARG(M == (int64_t)B * h * w, "conv_proj_dw: x has %lld rows, %lld expected", (long long)M,
                 (long long)B * h * w);
  B200_CHECK_ARG(aligned16(x) && aligned16(wq) && aligned16(bq) && aligned16(wkv) && aligned16(bkv) &&
                     aligned16(q_out) && aligned16(kv_out),
                 "conv_proj_dw: pointers must be 16-byte aligned");
  const int oh = (h - 1) / s + 1, ow = (w - 1) / s + 1;
  const long long bytes_x = M * C * 2, bytes_kv = (long long)B * oh * ow * C * 2;
  B200_CHECK_ARG(!overlap(x, bytes_x, q_out, bytes_x) && !overlap(x, bytes_x, kv_out, bytes_kv),
                 "conv_proj_dw: x must overlap neither output (every token reads its neighbours)");
  const long long total8 = M * (C / 8);
  B200_CHECK_ARG((total8 + CP_THREADS - 1) / CP_THREADS <= 0x7fffffffLL, "conv_proj_dw: %lld elements exceed the grid",
                 total8 * 8);
  auto kern = k == 1 ? conv_proj_dw_kernel<1> : k == 3 ? conv_proj_dw_kernel<3> : k == 5 ? conv_proj_dw_kernel<5>
                                                                                         : conv_proj_dw_kernel<7>;
  kern<<<(unsigned)((total8 + CP_THREADS - 1) / CP_THREADS), CP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), wq, bq, wkv, bkv, reinterpret_cast<__nv_bfloat16*>(q_out),
      reinterpret_cast<__nv_bfloat16*>(kv_out), total8, h, w, oh, ow, C, s);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
