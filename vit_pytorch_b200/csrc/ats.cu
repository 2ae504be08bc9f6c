// The operations of Adaptive Token Sampling (reference ats_vit.py) that no other kernel covers.
//
// b200vit_ats_select: one CTA per image on the layer's packed qkv.  It decides whether the layer samples (the padded
//   length of the whole batch, max_b L_b, minus the cls token exceeds K: ats_vit.py:169), and if so computes the cls
//   query's softmax over the image's L_b valid keys per head in fp32, the value-norm weighted scores summed over the
//   heads, their normalised logarithm (ats_vit.py:51-75), and K Gumbel-max draws over them (ats_vit.py:79-87).  The
//   drawn ids are kept once each, sorted, behind the cls row (torch.unique + pad_sequence + F.pad, ats_vit.py:91-103).
//   Out: the row map src (padding rows point at the image's cls row), the new valid lengths and the token ids carried
//   along (ats_vit.py:161-163).  A layer that does not sample writes the identity map.
// b200vit_ats_gather: out rows = in rows src[r], fp32 stream and/or a bf16 column range, as bit copies.
// The attention of the kept queries is b200vit_attention_kv_lens (twins.cu).
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int ATS_THREADS = 256;
constexpr int ATS_WARPS = ATS_THREADS / 32;
constexpr float ATS_EPS = 1e-6f;  // AdaptiveTokenSampling's eps and sample_gumbel's (ats_vit.py:19-25, 45)

struct AtsParams {
  const __nv_bfloat16* qkv;
  long long ld;
  const int* len_in;
  const int* ids_in;
  const void* u;
  int u_bf16;
  int* src;
  int* len_out;
  int* ids_out;
  int B, S_in, S_out, K, H, dh;
  float scale;
};

// torch.argmax order: a NaN beats every number and the first NaN wins; among numbers the larger, ties to the lower index
__device__ __forceinline__ bool ats_better(float a, int ia, float b, int ib) {
  const bool na = isnan(a), nb = isnan(b);
  if (na || nb) return na && (!nb || ia < ib);
  return a > b || (a == b && ia < ib);
}

__device__ __forceinline__ float ats_uniform(const AtsParams& p, long long i) {
  return p.u_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.u)[i])
                  : reinterpret_cast<const float*>(p.u)[i];
}

__global__ void __launch_bounds__(ATS_THREADS) ats_select_kernel(const AtsParams p) {
  extern __shared__ float ats_smem[];
  __shared__ float red[ATS_WARPS];
  __shared__ int ired[ATS_WARPS];
  __shared__ int s_kept;
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int S = p.S_in, H = p.H, dh = p.dh;

  // the batch's padded length decides for every image
  int mx = 0;
  for (int i = tid; i < p.B; i += ATS_THREADS) mx = max(mx, p.len_in[i]);
  for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) ired[warp] = mx;
  __syncthreads();
  mx = ired[0];
  for (int w = 1; w < ATS_WARPS; ++w) mx = max(mx, ired[w]);
  const int L = min(max(p.len_in[b], 1), S);
  const int* ids_in = p.ids_in + (long long)b * S;
  int* src = p.src + (long long)b * p.S_out;
  int* ids_out = p.ids_out + (long long)b * p.S_out;

  if (!(mx - 1 > p.K)) {  // no sampling: the identity map (L <= K + 1 <= S_out)
    for (int r = tid; r < p.S_out; r += ATS_THREADS) {
      const int pr = r < L ? r : 0;
      src[r] = b * S + pr;
      ids_out[r] = ids_in[pr];
    }
    if (tid == 0) p.len_out[b] = L;
    return;
  }

  float* d = ats_smem;                    // [H][S] scale * q_cls . k_j
  float* vn = d + (size_t)H * S;          // [H][S] |v_j| per head
  float* sc = vn + (size_t)H * S;         // [S] the scores s_j, then the pseudo-logits (candidate c = j - 1 at c)
  float* hmax = sc + S;                   // [H]
  float* hsum = hmax + H;                 // [H]
  int* pos = reinterpret_cast<int*>(hsum + H);            // [S] kept positions, cls first
  unsigned char* chosen = reinterpret_cast<unsigned char*>(pos + S);  // [S]

  const __nv_bfloat16* base = p.qkv + (long long)b * S * p.ld;
  const int I = H * dh;
  for (int t = tid; t < H * L; t += ATS_THREADS) {
    const int j = t / H, h = t - j * H;
    const uint4* q = reinterpret_cast<const uint4*>(base + h * dh);
    const uint4* k = reinterpret_cast<const uint4*>(base + (long long)j * p.ld + I + h * dh);
    const uint4* v = reinterpret_cast<const uint4*>(base + (long long)j * p.ld + 2 * I + h * dh);
    float dot = 0.f, nv = 0.f;
    for (int c = 0; c < dh / 8; ++c) {
      const uint4 qa = q[c], ka = k[c], va = v[c];
      const uint32_t qw[4] = {qa.x, qa.y, qa.z, qa.w}, kw[4] = {ka.x, ka.y, ka.z, ka.w}, vw[4] = {va.x, va.y, va.z, va.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {  // a bf16 pair as two exact fp32 values: the low half first
        dot = fmaf(__uint_as_float(qw[e] << 16), __uint_as_float(kw[e] << 16), dot);
        dot = fmaf(__uint_as_float(qw[e] & 0xffff0000u), __uint_as_float(kw[e] & 0xffff0000u), dot);
        nv = fmaf(__uint_as_float(vw[e] << 16), __uint_as_float(vw[e] << 16), nv);
        nv = fmaf(__uint_as_float(vw[e] & 0xffff0000u), __uint_as_float(vw[e] & 0xffff0000u), nv);
      }
    }
    d[h * S + j] = dot * p.scale;
    vn[h * S + j] = sqrtf(nv);
  }
  if (tid == 0) s_kept = 0;
  for (int j = tid; j < S; j += ATS_THREADS) chosen[j] = 0;
  __syncthreads();

  // per head: the softmax's max and sum over the L valid keys (the cls key included, ats_vit.py:146)
  for (int h = warp; h < H; h += ATS_WARPS) {
    float m = -INFINITY;
    for (int j = lane; j < L; j += 32) m = fmaxf(m, d[h * S + j]);
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < L; j += 32) s += expf(d[h * S + j] - m);
    s = warp_sum(s);
    if (lane == 0) {
      hmax[h] = m;
      hsum[h] = s;
    }
  }
  __syncthreads();

  // s_j = sum_h p_h[j] |v_h,j| for j >= 1 (ats_vit.py:57-63) and its total
  float part = 0.f;
  for (int j = 1 + tid; j < L; j += ATS_THREADS) {
    float s = 0.f;
    for (int h = 0; h < H; ++h) s += expf(d[h * S + j] - hmax[h]) / hsum[h] * vn[h * S + j];
    part += s;
    sc[j - 1] = s;
  }
  part = warp_sum(part);
  if (lane == 0) red[warp] = part;
  __syncthreads();
  float total = 0.f;
  for (int w = 0; w < ATS_WARPS; ++w) total += red[w];
  // pseudo-logits log(s_j / (total + eps) + eps) (ats_vit.py:67-71)
  for (int c = tid; c < L - 1; c += ATS_THREADS) sc[c] = logf(sc[c] / (total + ATS_EPS) + ATS_EPS);
  __syncthreads();

  // K Gumbel-max draws, one warp each: argmax_c (logit_c - log(-log(u + eps) + eps)) (ats_vit.py:21-25, 83-87)
  const long long urow = (long long)(S - 1);
  for (int k = warp; k < p.K; k += ATS_WARPS) {
    const long long u0 = ((long long)b * p.K + k) * urow;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < L - 1; c += 32) {
      const float u = ats_uniform(p, u0 + c);
      const float g = -logf(-logf(u + ATS_EPS) + ATS_EPS);
      const float v = sc[c] + g;
      if (ats_better(v, c, best, bi)) {
        best = v;
        bi = c;
      }
    }
    for (int o = 16; o; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ats_better(ov, oi, best, bi)) {
        best = ov;
        bi = oi;
      }
    }
    if (lane == 0 && bi < L - 1) chosen[bi] = 1;
  }
  __syncthreads();

  // sorted unique positions behind the cls row
  if (warp == 0) {
    int count = 0;
    for (int c0 = 0; c0 < L - 1; c0 += 32) {
      const int c = c0 + lane;
      const bool f = c < L - 1 && chosen[c];
      const unsigned m = __ballot_sync(0xffffffffu, f);
      if (f) pos[1 + count + __popc(m & ((1u << lane) - 1u))] = c + 1;
      count += __popc(m);
    }
    if (lane == 0) {
      pos[0] = 0;
      s_kept = count;
    }
  }
  __syncthreads();
  const int kept = s_kept;
  for (int r = tid; r < p.S_out; r += ATS_THREADS) {
    const int pr = r <= kept ? pos[r] : 0;
    src[r] = b * S + pr;
    ids_out[r] = ids_in[pr];
  }
  if (tid == 0) p.len_out[b] = 1 + kept;
}

size_t ats_select_smem(int S, int H) { return (size_t)H * S * 8 + (size_t)H * 8 + (size_t)S * 9 + 16; }

// one warp per output row: fp32 x row (float4) and bf16 column range (uint4)
__global__ void __launch_bounds__(256)
ats_gather_kernel(const int* __restrict__ src, int rows, const float* __restrict__ x, long long ldx,
                  float* __restrict__ xo, long long ldxo, int D, const __nv_bfloat16* __restrict__ a, long long lda,
                  __nv_bfloat16* __restrict__ ao, long long ldao, int ncols) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const long long s = src[r];
  if (x) {
    const float4* in = reinterpret_cast<const float4*>(x + s * ldx);
    float4* out = reinterpret_cast<float4*>(xo + (long long)r * ldxo);
    for (int c = lane; c < D / 4; c += 32) out[c] = in[c];
  }
  if (a) {
    const uint4* in = reinterpret_cast<const uint4*>(a + s * lda);
    uint4* out = reinterpret_cast<uint4*>(ao + (long long)r * ldao);
    for (int c = lane; c < ncols / 8; c += 32) out[c] = in[c];
  }
}

}  // namespace b200

using namespace b200;

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int b200vit_ats_select(const void* qkv, int64_t ld, const int32_t* len_in, const int32_t* ids_in,
                                  const void* u, int u_bf16, int32_t* src, int32_t* len_out, int32_t* ids_out, int B,
                                  int S_in, int S_out, int K, int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(qkv && len_in && ids_in && u && src && len_out && ids_out, "ats_select: null pointer");
  B200_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && K > 0, "ats_select: bad shape B=%d H=%d K=%d", B, H, K);
  B200_CHECK_ARG(S_in >= 2 && S_in <= B200VIT_ATS_MAX_TOKENS, "ats_select: S_in=%d outside [2, %d]", S_in,
                 B200VIT_ATS_MAX_TOKENS);
  B200_CHECK_ARG((long long)H * S_in <= B200VIT_ATS_MAX_HEAD_TOKENS, "ats_select: H * S_in = %lld > %d",
                 (long long)H * S_in, B200VIT_ATS_MAX_HEAD_TOKENS);
  B200_CHECK_ARG(S_out == (S_in < K + 1 ? S_in : K + 1), "ats_select: S_out=%d must be min(S_in, K + 1) = %d", S_out,
                 S_in < K + 1 ? S_in : K + 1);
  B200_CHECK_ARG(head_width_ok(dh), "ats_select: dim_head=%d not supported by this build (32, 64, 80 or 128)", dh);
  B200_CHECK_ARG(ld >= 3LL * H * dh && ld % 8 == 0, "ats_select: ld=%lld must be a multiple of 8 and >= %d",
                 (long long)ld, 3 * H * dh);
  B200_CHECK_ARG(aligned16(qkv), "ats_select: qkv must be 16-byte aligned");
  B200_CHECK_ARG(len_in != len_out && ids_in != ids_out, "ats_select: lengths and ids cannot be updated in place");
  AtsParams p{};
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv);
  p.ld = ld;
  p.len_in = len_in;
  p.ids_in = ids_in;
  p.u = u;
  p.u_bf16 = u_bf16 ? 1 : 0;
  p.src = src;
  p.len_out = len_out;
  p.ids_out = ids_out;
  p.B = B;
  p.S_in = S_in;
  p.S_out = S_out;
  p.K = K;
  p.H = H;
  p.dh = dh;
  p.scale = scale;
  const size_t bytes = ats_select_smem(S_in, H);
  B200_ENSURE_SMEM(ats_select_kernel, bytes);
  ats_select_kernel<<<B, ATS_THREADS, bytes, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_ats_gather(const int32_t* src, int rows, const float* x, int64_t ldx, float* x_out,
                                  int64_t ldx_out, int D, const void* a, int64_t lda, void* a_out, int64_t lda_out,
                                  int ncols, void* stream) {
  B200_CHECK_ARG(src && rows > 0, "ats_gather: null row map or rows=%d", rows);
  B200_CHECK_ARG((x != nullptr) == (x_out != nullptr) && (a != nullptr) == (a_out != nullptr) && (x || a),
                 "ats_gather: give x with x_out and/or a with a_out");
  if (x) {
    B200_CHECK_ARG(D > 0 && D % 4 == 0 && ldx % 4 == 0 && ldx_out % 4 == 0 && ldx >= D && ldx_out >= D,
                   "ats_gather: D=%d, ldx=%lld, ldx_out=%lld must be multiples of 4 with ld >= D", D, (long long)ldx,
                   (long long)ldx_out);
    B200_CHECK_ARG(aligned16(x) && aligned16(x_out), "ats_gather: x and x_out must be 16-byte aligned");
    B200_CHECK_ARG(x != x_out, "ats_gather: x_out cannot be x (rows of other CTAs would be overwritten)");
  }
  if (a) {
    B200_CHECK_ARG(ncols > 0 && ncols % 8 == 0 && lda % 8 == 0 && lda_out % 8 == 0 && lda >= ncols &&
                       lda_out >= ncols,
                   "ats_gather: ncols=%d, lda=%lld, lda_out=%lld must be multiples of 8 with ld >= ncols", ncols,
                   (long long)lda, (long long)lda_out);
    B200_CHECK_ARG(aligned16(a) && aligned16(a_out) && a != a_out, "ats_gather: a and a_out must be 16-byte aligned "
                   "and distinct");
  }
  ats_gather_kernel<<<(rows + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, rows, x, ldx, x_out, ldx_out, D, reinterpret_cast<const __nv_bfloat16*>(a), lda,
      reinterpret_cast<__nv_bfloat16*>(a_out), lda_out, ncols);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
