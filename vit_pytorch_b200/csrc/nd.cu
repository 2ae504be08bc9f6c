// The N-dimensional ViTs (reference vit_nd.py / vit_nd_rotary.py): the patch gather of an input of any rank 1..7 and
// the golden-gate rotary embedding of q and k.  Both are HBM-bound bit movers around the GEMMs.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------------------------
// N-d patchify: img[B, C, S_0 .. S_{r-1}] -> A[B*n, ldo],
//   A[b*n + rowmajor(g), rowmajor(q)*C + c] = img[b, c, g_0*p_0 + q_0, ..., g_{r-1}*p_{r-1} + q_{r-1}]
// the einops pattern 'b c (f p0) (g p1) ... -> b (f g ...) (p0 p1 ... c)' of vit_nd.py:130-142 / vit_nd_rotary.py:216-228.
// One CTA per (image, patch coordinates g_0..g_{r-2}, run of `wc` patches along the last axis).  The C x (p_0 .. p_{r-2})
// input rows of that run are contiguous along the last axis: they are staged in shared memory with coalesced loads
// (16 bytes wide when the rows allow), then every thread assembles 8 consecutive output columns and stores them as one
// 16-byte word.  Columns [K, ldo) are written as zeros (K padding of the GEMM's A operand).
// ---------------------------------------------------------------------------------------------------------------
struct NdGeom {
  int rank, C;
  int G[7], p[7];            // patches per axis, patch extent per axis
  long long stride[7];       // element stride of axis i inside one channel
  long long chan;            // elements per channel
  int K;                     // patch_dim = C * prod(p)
  int Pp;                    // prod(p_0 .. p_{r-2})
  int Gp;                    // prod(G_0 .. G_{r-2})
  int n;                     // patches per image
  int wc, nchunk;            // last-axis patches per CTA, CTAs along the last axis
};

__global__ void __launch_bounds__(256)
patchify_nd_kernel(const __nv_bfloat16* __restrict__ img, __nv_bfloat16* __restrict__ out, long long ldo, NdGeom g,
                   int vec) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int last = g.rank - 1;
  const int pl = g.p[last];
  const int rows = g.C * g.Pp;
  long long* roff = reinterpret_cast<long long*>(smem_raw);                      // [rows] input row offsets
  uint16_t* slab = reinterpret_cast<uint16_t*>(smem_raw + ((size_t)rows * 8 + 15) / 16 * 16);  // [rows][L]
  long long item = blockIdx.x;
  const int chunk = (int)(item % g.nchunk);
  item /= g.nchunk;
  const int gp = (int)(item % g.Gp);
  const long long b = item / g.Gp;
  const int g0 = chunk * g.wc;
  const int wc = min(g.wc, g.G[last] - g0);
  const int L = wc * pl;
  long long base = b * g.C * g.chan + (long long)g0 * pl;
  {
    int rem = gp;
    for (int i = last - 1; i >= 0; --i) {
      const int gi = rem % g.G[i];
      rem /= g.G[i];
      base += (long long)gi * g.p[i] * g.stride[i];
    }
  }
  for (int row = threadIdx.x; row < rows; row += blockDim.x) {
    const int c = row / g.Pp;
    int rem = row - c * g.Pp;
    long long off = (long long)c * g.chan;
    for (int i = last - 1; i >= 0; --i) {
      const int qi = rem % g.p[i];
      rem /= g.p[i];
      off += (long long)qi * g.stride[i];
    }
    roff[row] = base + off;
  }
  __syncthreads();
  if (vec) {
    const int vpr = L >> 3;
    for (int i = threadIdx.x; i < rows * vpr; i += blockDim.x) {
      const int row = i / vpr, v = i - row * vpr;
      const uint4 w = __ldg(reinterpret_cast<const uint4*>(img + roff[row]) + v);
      *reinterpret_cast<uint4*>(slab + (size_t)row * L + 8 * v) = w;
    }
  } else {
    const uint16_t* src = reinterpret_cast<const uint16_t*>(img);
    for (int i = threadIdx.x; i < rows * L; i += blockDim.x) {
      const int row = i / L, x = i - row * L;
      slab[i] = src[roff[row] + x];
    }
  }
  __syncthreads();
  const int vpo = (int)(ldo >> 3);
  __nv_bfloat16* obase = out + (b * g.n + (long long)gp * g.G[last] + g0) * ldo;
  for (int j = threadIdx.x; j < wc * vpo; j += blockDim.x) {
    const int rl = j / vpo, e0 = (j - rl * vpo) * 8;
    // column e = (qp*pl + ql)*C + c, walked in order from e0
    int c = e0 % g.C, qi = e0 / g.C;
    int ql = qi % pl, qp = qi / pl;
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 8; k += 2) {
      uint32_t lo = 0u, hi = 0u;
      if (e0 + k < g.K) lo = slab[(size_t)(c * g.Pp + qp) * L + rl * pl + ql];
      if (++c == g.C) { c = 0; if (++ql == pl) { ql = 0; ++qp; } }
      if (e0 + k + 1 < g.K) hi = slab[(size_t)(c * g.Pp + qp) * L + rl * pl + ql];
      if (++c == g.C) { c = 0; if (++ql == pl) { ql = 0; ++qp; } }
      w[k >> 1] = lo | (hi << 16);
    }
    *reinterpret_cast<uint4*>(obase + (long long)rl * ldo + e0) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Golden-gate N-d rotary embedding of q and k, in place on qkv[T, 3*H*DH] (GoldenGateRoPENd.forward,
// vit_nd_rotary.py:74-96).  One thread per (token, head, 8 frequencies): it reads the 8 (cos, sin) pairs once and
// rotates the same frequencies of q and of k.  Every product and sum is rounded on its own (no FMA contraction), the
// operation order of the reference's fp32 expression, so the result is bit-identical to it for the same table.
// ---------------------------------------------------------------------------------------------------------------
template <int DH>
__global__ void __launch_bounds__(256)
rope_qk_kernel(__nv_bfloat16* __restrict__ qkv, const float* __restrict__ cs, int R, long long T, int H) {
  constexpr int HALF = DH / 2, CH = HALF / 8;
  const long long item = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= T * H * CH) return;
  const int ch = (int)(item % CH);
  const long long th = item / CH;
  const int h = (int)(th % H);
  const long long t = th / H;
  const int f0 = ch * 8;
  const float4* c4 = reinterpret_cast<const float4*>(cs + ((t % R) * H + h) * DH + 2 * f0);  // [R][H][HALF][2]
  float cth[8], sth[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 v = __ldg(c4 + i);
    cth[2 * i] = v.x;
    sth[2 * i] = v.y;
    cth[2 * i + 1] = v.z;
    sth[2 * i + 1] = v.w;
  }
#pragma unroll
  for (int s = 0; s < 2; ++s) {  // q, then k
    __nv_bfloat16* hp = qkv + t * 3 * H * DH + (long long)s * H * DH + (long long)h * DH + f0;
    const uint4 xr = *reinterpret_cast<const uint4*>(hp);
    const uint4 yr = *reinterpret_cast<const uint4*>(hp + HALF);
    const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(&xr);
    const __nv_bfloat162* y2 = reinterpret_cast<const __nv_bfloat162*>(&yr);
    uint32_t xo[4], yo[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = __bfloat1622float2(x2[i]), y = __bfloat1622float2(y2[i]);
      const float c0 = cth[2 * i], s0 = sth[2 * i], c1 = cth[2 * i + 1], s1 = sth[2 * i + 1];
      xo[i] = pack_bf16x2(__fsub_rn(__fmul_rn(x.x, c0), __fmul_rn(y.x, s0)),
                          __fsub_rn(__fmul_rn(x.y, c1), __fmul_rn(y.y, s1)));
      yo[i] = pack_bf16x2(__fadd_rn(__fmul_rn(x.x, s0), __fmul_rn(y.x, c0)),
                          __fadd_rn(__fmul_rn(x.y, s1), __fmul_rn(y.y, c1)));
    }
    *reinterpret_cast<uint4*>(hp) = make_uint4(xo[0], xo[1], xo[2], xo[3]);
    *reinterpret_cast<uint4*>(hp + HALF) = make_uint4(yo[0], yo[1], yo[2], yo[3]);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200vit_patchify_nd(const void* img, void* out_bf16, int64_t ldo, int B, int C, int rank,
                                   const int* shape, const int* patch, void* stream) {
  B200_CHECK_ARG(img && out_bf16 && shape && patch, "patchify_nd: null pointer");
  B200_CHECK_ARG(rank >= 1 && rank <= 7, "patchify_nd: rank %d outside 1..7", rank);
  B200_CHECK_ARG(B > 0 && C > 0, "patchify_nd: bad shape B=%d C=%d", B, C);
  NdGeom g{};
  g.rank = rank;
  g.C = C;
  long long K = C, n = 1, Pp = 1, Gp = 1, chan = 1;
  for (int i = rank - 1; i >= 0; --i) {
    B200_CHECK_ARG(shape[i] > 0 && patch[i] > 0 && shape[i] % patch[i] == 0,
                   "patchify_nd: axis %d of extent %d not divisible by patch %d", i, shape[i], patch[i]);
    g.stride[i] = chan;
    chan *= shape[i];
    g.p[i] = patch[i];
    g.G[i] = shape[i] / patch[i];
    K *= patch[i];
    n *= g.G[i];
    if (i < rank - 1) {
      Pp *= patch[i];
      Gp *= g.G[i];
    }
  }
  B200_CHECK_ARG(ldo % 8 == 0 && ldo >= K, "patchify_nd: ldo=%lld must be a multiple of 8 and >= patch_dim %lld",
                 (long long)ldo, K);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0 && (reinterpret_cast<uintptr_t>(img) & 1) == 0,
                 "patchify_nd: misaligned pointer (out needs 16 bytes, img 2)");
  B200_CHECK_ARG(n * B < (1ll << 31) && K < (1 << 30), "patchify_nd: too many patches");
  g.chan = chan;
  g.K = (int)K;
  g.Pp = (int)Pp;
  g.Gp = (int)Gp;
  g.n = (int)n;
  const int pl = patch[rank - 1], Gl = g.G[rank - 1];
  // ~32 KB of staged input per CTA; runs of a multiple of 8 / gcd(pl, 8) patches keep the rows 16-byte sized
  int wc = (int)(16384 / K);
  const int m = 8 / ((pl & 7) == 0 ? 8 : (pl & 3) == 0 ? 4 : (pl & 1) == 0 ? 2 : 1);
  if (wc >= Gl) wc = Gl;
  else if (wc >= m) wc -= wc % m;
  else if (wc < 1) wc = 1;
  g.wc = wc;
  g.nchunk = (Gl + wc - 1) / wc;
  const size_t smem = ((size_t)C * Pp * 8 + 15) / 16 * 16 + (size_t)wc * K * 2;
  B200_CHECK_ARG(smem <= 200 * 1024, "patchify_nd: a patch of %lld elements exceeds shared memory", K);
  const int vec = shape[rank - 1] % 8 == 0 && (wc * pl) % 8 == 0 && (reinterpret_cast<uintptr_t>(img) & 15) == 0;
  B200_ENSURE_SMEM(patchify_nd_kernel, smem);
  const long long blocks = (long long)B * Gp * g.nchunk;
  B200_CHECK_ARG(blocks < (1ll << 31), "patchify_nd: too many patches");
  patchify_nd_kernel<<<(unsigned)blocks, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(img), reinterpret_cast<__nv_bfloat16*>(out_bf16), (long long)ldo, g, vec);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_rope_qk(void* qkv, const float* cs, int R, int T, int H, int dh, void* stream) {
  B200_CHECK_ARG(qkv && cs, "rope_qk: null pointer");
  B200_CHECK_ARG(T > 0 && H > 0 && R > 0, "rope_qk: bad shape T=%d H=%d R=%d", T, H, R);
  B200_CHECK_ARG(head_width_ok(dh), "rope_qk: dim_head=%d not supported by this build (32, 64, 80 or 128)", dh);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(cs) & 15) == 0,
                 "rope_qk: qkv and cs must be 16-byte aligned");
  const long long threads = (long long)T * H * (dh / 16);
  const unsigned grid = (unsigned)((threads + 255) / 256);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  auto* q = reinterpret_cast<__nv_bfloat16*>(qkv);
  switch (dh) {
    case 32: rope_qk_kernel<32><<<grid, 256, 0, st>>>(q, cs, R, T, H); break;
    case 64: rope_qk_kernel<64><<<grid, 256, 0, st>>>(q, cs, R, T, H); break;
    case 80: rope_qk_kernel<80><<<grid, 256, 0, st>>>(q, cs, R, T, H); break;
    default: rope_qk_kernel<128><<<grid, 256, 0, st>>>(q, cs, R, T, H); break;
  }
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
