// Cross-covariance attention (XCiT's XCA, reference xcit.py:109-148): attention over the dh channels of a head instead
// of over its N tokens.  Per (image b, head h), with q, k, v the [N, dh] slices of the packed QKV projection:
//   G = q^T k (dh x dh),  sq_i = sum_n q_ni^2,  sk_j = sum_n k_nj^2
//   A_ij = softmax_j(tau_h G_ij / (max(sqrt(sq_i), 1e-12) max(sqrt(sk_j), 1e-12)))      (F.normalize's eps rule)
//   out_ni = sum_j A_ij v_nj
// The cost is linear in N and nothing N x N exists.  One CTA of 256 threads per (image, head), two passes over the
// tokens in tiles of T rows staged in shared memory as fp32:
//   pass 1: every thread owns an R x R block of G (R = dh / 16, rows ty + 16a, columns tx + 16c of a 16 x 16 thread
//           grid) and accumulates it on the CUDA cores; threads 0..dh-1 and 128..128+dh-1 accumulate the column sums of
//           squares of q and k from the same tiles.  Rows past N are zero-filled, so they add nothing.
//   softmax: row i of the scores lives in the 16 lanes of one half-warp; max and sum are butterfly reductions over
//           those lanes, and A goes to shared memory in fp32.
//   pass 2: every thread owns T / 16 token rows x R channels of the output tile O = V A^T and stores the rows below N.
// Accumulation, norms and softmax are fp32; there are no atomics and every sum has a fixed order, so repeated calls
// give the same bits.  Each CTA reads only its own image's rows.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

template <int DH>
struct XcaShape {
  static constexpr int R = DH / 16;               // G entries per thread along each axis
  static constexpr int T = DH >= 128 ? 32 : 64;   // tokens per tile (two CTAs per SM at dh 128)
  static constexpr int LDT = DH + 4;              // tile row stride (floats): keeps float4 stores, spreads banks
  static constexpr int LDA = DH + 1;              // A row stride: conflict-free column reads in pass 2
  static constexpr size_t smem = (size_t)(2 * T * LDT + DH * LDA + 2 * DH) * sizeof(float);
};

// rows [n0, n0 + T) of one dh-wide slice (column offset col) of the packed rows -> fp32 tile, zeros past N
template <int DH>
__device__ __forceinline__ void xca_stage(float* __restrict__ dst, const __nv_bfloat16* __restrict__ base, long long ld,
                                          int col, int n0, int N) {
  using S = XcaShape<DH>;
  constexpr int CH = DH / 8;                      // 16-byte chunks per row
  for (int e = threadIdx.x; e < S::T * CH; e += 256) {
    const int r = e / CH, c = e % CH;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (n0 + r < N) v = *reinterpret_cast<const uint4*>(base + (long long)(n0 + r) * ld + col + c * 8);
    float* d = dst + r * S::LDT + c * 8;
    *reinterpret_cast<float4*>(d) = make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xFFFF0000u),
                                                __uint_as_float(v.y << 16), __uint_as_float(v.y & 0xFFFF0000u));
    *reinterpret_cast<float4*>(d + 4) = make_float4(__uint_as_float(v.z << 16), __uint_as_float(v.z & 0xFFFF0000u),
                                                    __uint_as_float(v.w << 16), __uint_as_float(v.w & 0xFFFF0000u));
  }
}

template <int DH>
__global__ void __launch_bounds__(256)
xca_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ tau, __nv_bfloat16* __restrict__ out,
           int N, int H) {
  using S = XcaShape<DH>;
  constexpr int R = S::R, T = S::T, LDT = S::LDT, LDA = S::LDA, TA = T / 16;
  extern __shared__ float4 xca_smem4[];
  float* qs = reinterpret_cast<float*>(xca_smem4);   // [T][LDT]   pass 1: q tile; pass 2: v tile
  float* ks = qs + T * LDT;                          // [T][LDT]   pass 1: k tile
  float* as = ks + T * LDT;                          // [DH][LDA]  A
  float* rq = as + DH * LDA;                         // [DH]       1 / max(|q_i|, 1e-12)
  float* rk = rq + DH;                               // [DH]       1 / max(|k_j|, 1e-12)
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int I = H * DH;
  const long long ld = 3LL * I;
  const __nv_bfloat16* base = qkv + (long long)b * N * ld + h * DH;

  // ---- pass 1: G = q^T k and the column sums of squares
  float g[R][R];
#pragma unroll
  for (int a = 0; a < R; ++a)
#pragma unroll
    for (int c = 0; c < R; ++c) g[a][c] = 0.f;
  float ss = 0.f;
  const float* sqcol = tid < DH ? qs + tid : (tid >= 128 && tid < 128 + DH ? ks + (tid - 128) : nullptr);
  for (int n0 = 0; n0 < N; n0 += T) {
    xca_stage<DH>(qs, base, ld, 0, n0, N);
    xca_stage<DH>(ks, base, ld, I, n0, N);
    __syncthreads();
#pragma unroll 4
    for (int n = 0; n < T; ++n) {
      float qa[R], kc[R];
#pragma unroll
      for (int a = 0; a < R; ++a) qa[a] = qs[n * LDT + ty + 16 * a];
#pragma unroll
      for (int c = 0; c < R; ++c) kc[c] = ks[n * LDT + tx + 16 * c];
#pragma unroll
      for (int a = 0; a < R; ++a)
#pragma unroll
        for (int c = 0; c < R; ++c) g[a][c] = fmaf(qa[a], kc[c], g[a][c]);
    }
    if (sqcol != nullptr) {
#pragma unroll 8
      for (int n = 0; n < T; ++n) {
        const float v = sqcol[n * LDT];
        ss = fmaf(v, v, ss);
      }
    }
    __syncthreads();
  }
  if (tid < DH) rq[tid] = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
  else if (tid >= 128 && tid < 128 + DH) rk[tid - 128] = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
  __syncthreads();

  // ---- softmax over j of tau * G_ij / (|q_i| |k_j|); row i = ty + 16a lives in the half-warp of lanes with this ty
  const float t = tau[h];
  float rkc[R];
#pragma unroll
  for (int c = 0; c < R; ++c) rkc[c] = rk[tx + 16 * c];
#pragma unroll
  for (int a = 0; a < R; ++a) {
    const float sa = t * rq[ty + 16 * a];
    float m = -INFINITY;
#pragma unroll
    for (int c = 0; c < R; ++c) {
      g[a][c] = sa * g[a][c] * rkc[c];
      m = fmaxf(m, g[a][c]);
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float l = 0.f;
#pragma unroll
    for (int c = 0; c < R; ++c) {
      g[a][c] = expf(g[a][c] - m);
      l += g[a][c];
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
    const float inv = 1.0f / l;
#pragma unroll
    for (int c = 0; c < R; ++c) as[(ty + 16 * a) * LDA + tx + 16 * c] = g[a][c] * inv;
  }
  __syncthreads();

  // ---- pass 2: O = V A^T, tile by tile
  __nv_bfloat16* ob = out + (long long)b * N * I + h * DH;
  for (int n0 = 0; n0 < N; n0 += T) {
    xca_stage<DH>(qs, base, ld, 2 * I, n0, N);
    __syncthreads();
    float acc[TA][R];
#pragma unroll
    for (int a = 0; a < TA; ++a)
#pragma unroll
      for (int c = 0; c < R; ++c) acc[a][c] = 0.f;
#pragma unroll 4
    for (int j = 0; j < DH; ++j) {
      float va[TA], ac[R];
#pragma unroll
      for (int a = 0; a < TA; ++a) va[a] = qs[(ty + 16 * a) * LDT + j];
#pragma unroll
      for (int c = 0; c < R; ++c) ac[c] = as[(tx + 16 * c) * LDA + j];
#pragma unroll
      for (int a = 0; a < TA; ++a)
#pragma unroll
        for (int c = 0; c < R; ++c) acc[a][c] = fmaf(va[a], ac[c], acc[a][c]);
    }
#pragma unroll
    for (int a = 0; a < TA; ++a) {
      const int n = n0 + ty + 16 * a;
      if (n < N) {
#pragma unroll
        for (int c = 0; c < R; ++c) ob[(long long)n * I + tx + 16 * c] = __float2bfloat16_rn(acc[a][c]);
      }
    }
    __syncthreads();
  }
}

template <int DH>
static int launch_xca(const void* qkv, const float* tau, void* out, int B, int N, int H, cudaStream_t st) {
  const size_t smem = XcaShape<DH>::smem;
  B200_ENSURE_SMEM(xca_kernel<DH>, smem);
  xca_kernel<DH><<<B * H, 256, smem, st>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), tau,
                                            reinterpret_cast<__nv_bfloat16*>(out), N, H);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" int b200vit_attention_xca(const void* qkv, const float* tau, void* out, int B, int N, int H, int dh,
                                     void* stream) {
  B200_CHECK_ARG(qkv && tau && out, "attention_xca: null pointer");
  B200_CHECK_ARG(B > 0 && N > 0 && H > 0, "attention_xca: bad shape B=%d N=%d H=%d", B, N, H);
  B200_CHECK_ARG(dh == 32 || dh == 48 || dh == 64 || dh == 80 || dh == 128,
                 "attention_xca: dim_head=%d not supported by this build (32, 48, 64, 80 or 128)", dh);
  B200_CHECK_ARG(N <= 16384, "attention_xca: N=%d exceeds 16384 tokens", N);
  B200_CHECK_ARG(((int64_t)H * dh) % 8 == 0, "attention_xca: H*dim_head=%lld must be a multiple of 8",
                 (long long)H * dh);
  B200_CHECK_ARG((int64_t)B * H <= 0x7fffffff, "attention_xca: B*H too large");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "attention_xca: qkv and out must be 16-byte aligned");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(tau) & 3) == 0, "attention_xca: tau must be 4-byte aligned");
  auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: return launch_xca<32>(qkv, tau, out, B, N, H, st);
    case 48: return launch_xca<48>(qkv, tau, out, B, N, H, st);
    case 64: return launch_xca<64>(qkv, tau, out, B, N, H, st);
    case 80: return launch_xca<80>(qkv, tau, out, B, N, H, st);
    default: return launch_xca<128>(qkv, tau, out, B, N, H, st);
  }
}
