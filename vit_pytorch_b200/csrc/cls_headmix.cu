// Class-token attention with talking heads, for sm_90a (CaiT's class attention, reference cait.py:83-103 with a
// context): b200vit_attention_cls_headmix.  The query of image b is row b of qkv_self[B, 3 I] (q | k | v of LN(cls),
// I = H dh); its keys are its own k followed by n context rows (k | v, strided, as b200vit_attention_cls).  Per head:
//   s_h[j] = scale q_h . k_h[j];  s'_g = sum_h pre[h][g] s_h;  p_g = softmax_j(s'_g);  p'_f = sum_g post[g][f] p_g;
//   out_f = sum_j p'_f[j] v_f[j]
// Every output head depends on every head's score at each key, so one CTA of 8 warps owns all heads of one image:
//   pass 1  lane = key (keys 32 w + l, then + 256, ...): the H scores of the key (q in fp32 shared memory, the key row
//           read as 16-byte vectors), pre-mixed; online max / sum per (lane, mixed head), merged over lanes and warps
//           into a log2-sum-exp per head
//   pass 2  the same keys: exact p_g, post-mixed into p'_f, staged per warp in shared memory; then the warp walks its
//           32 keys with lane = 8-element slice of v (coalesced rows) and accumulates p'_f[j] v_f[j]; the 8 warps'
//           partial outputs are summed in shared memory.
// Softmax and both mixes are fp32.  dh = 32, 48, 64, 80, 128, H <= 16, H dh <= 1024, n = 0..16384.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int CH_THREADS = 256;
constexpr int CH_WARPS = CH_THREADS / 32;
constexpr int CH_HEADS = 16;
constexpr int CH_MAX_INNER = 1024;
constexpr int CH_SLICES = CH_MAX_INNER / (8 * 32);  // 8-element slices of a row per lane

struct ClsHeadmixParams {
  const __nv_bfloat16* self;  // [B][3 I]
  const __nv_bfloat16* ctx;   // [k | v] rows, image b's j-th at (b ctx_rows + ctx_first + j) ctx_ld
  long long ctx_ld, ctx_rows, ldo;
  int ctx_first, n;
  __nv_bfloat16* out;
  const float* pre;           // [H][H], [input head][output head]
  const float* post;
  int H, I;
  float scale_log2e;
};

// shared-memory load the compiler may not hoist out of the key loop (2 H^2 mixing weights would not fit registers)
__device__ __forceinline__ float lds_keep_cls(const float* p) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(smem_u32(p)));
  return v;
}

template <int DH>
__global__ void __launch_bounds__(CH_THREADS) attention_cls_headmix_kernel(const ClsHeadmixParams p) {
  static_assert(DH % 8 == 0 && DH <= 128, "dim_head");
  __shared__ __align__(16) float q_s[CH_MAX_INNER];                 // q scale log2(e)
  __shared__ float pre_s[CH_HEADS * CH_HEADS], post_s[CH_HEADS * CH_HEADS];   // zero-padded beyond H
  __shared__ float m_s[CH_WARPS][CH_HEADS], l_s[CH_WARPS][CH_HEADS], lse_s[CH_HEADS];
  // pass 2: p'[warp][f][32 keys], then the warps' partial outputs [warp][I]
  __shared__ __align__(16) float buf[CH_WARPS * CH_MAX_INNER];

  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = p.H, I = p.I, nk = p.n + 1;
  const __nv_bfloat16* self = p.self + (long long)b * 3 * I;
  for (int i = tid; i < I; i += CH_THREADS) q_s[i] = __bfloat162float(self[i]) * p.scale_log2e;
  for (int i = tid; i < CH_HEADS * CH_HEADS; i += CH_THREADS) {
    const int r = i / CH_HEADS, c = i % CH_HEADS;
    const bool in = r < H && c < H;
    pre_s[i] = in ? p.pre[r * H + c] : 0.f;
    post_s[i] = in ? p.post[r * H + c] : 0.f;
  }
  __syncthreads();

  // key j: 0 = the query token's own k (kv_include_self: LN(cls) is the first context row), j >= 1: context row j - 1.
  // v follows k at +I in both layouts
  auto key_row = [&](int j) -> const __nv_bfloat16* {
    return j == 0 ? self + I : p.ctx + ((long long)b * p.ctx_rows + p.ctx_first + j - 1) * p.ctx_ld;
  };
  // pre-mixed scores of key row k in log2 units; heads >= H are 0
  auto scores = [&](const __nv_bfloat16* k, float (&sm)[CH_HEADS]) {
    float s[CH_HEADS];
#pragma unroll
    for (int h = 0; h < CH_HEADS; ++h) {
      float acc = 0.f;
      if (h < H) {
#pragma unroll
        for (int c = 0; c < DH / 8; ++c) {
          const uint4 raw = __ldg(reinterpret_cast<const uint4*>(k + h * DH + 8 * c));
          const __nv_bfloat162* k2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
          const float4 qa = *reinterpret_cast<const float4*>(q_s + h * DH + 8 * c);
          const float4 qb = *reinterpret_cast<const float4*>(q_s + h * DH + 8 * c + 4);
          const float2 k0 = __bfloat1622float2(k2[0]), k1 = __bfloat1622float2(k2[1]);
          const float2 k2f = __bfloat1622float2(k2[2]), k3 = __bfloat1622float2(k2[3]);
          acc = fmaf(qa.x, k0.x, acc);
          acc = fmaf(qa.y, k0.y, acc);
          acc = fmaf(qa.z, k1.x, acc);
          acc = fmaf(qa.w, k1.y, acc);
          acc = fmaf(qb.x, k2f.x, acc);
          acc = fmaf(qb.y, k2f.y, acc);
          acc = fmaf(qb.z, k3.x, acc);
          acc = fmaf(qb.w, k3.y, acc);
        }
      }
      s[h] = acc;
    }
#pragma unroll
    for (int g = 0; g < CH_HEADS; ++g) sm[g] = 0.f;
#pragma unroll
    for (int h = 0; h < CH_HEADS; ++h)
#pragma unroll
      for (int g = 0; g < CH_HEADS; ++g) sm[g] = fmaf(lds_keep_cls(pre_s + h * CH_HEADS + g), s[h], sm[g]);
  };

  // ---- pass 1: per mixed head, max and sum of exp2 over all keys
  {
    float m[CH_HEADS], l[CH_HEADS];
#pragma unroll
    for (int g = 0; g < CH_HEADS; ++g) m[g] = -INFINITY, l[g] = 0.f;
    for (int j = 32 * warp + lane; j < nk; j += CH_THREADS) {
      float sm[CH_HEADS];
      scores(key_row(j), sm);
#pragma unroll
      for (int g = 0; g < CH_HEADS; ++g) {
        const float mn = fmaxf(m[g], sm[g]);
        l[g] = l[g] * fast_ex2(m[g] - mn) + fast_ex2(sm[g] - mn);   // m = -inf on the first key: exp2(-inf) = 0
        m[g] = mn;
      }
    }
#pragma unroll
    for (int g = 0; g < CH_HEADS; ++g) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m[g], o), l2 = __shfl_xor_sync(0xffffffffu, l[g], o);
        const float mn = fmaxf(m[g], m2);
        // lanes without a key hold (-inf, 0): their weight is 0, and two of them stay (-inf, 0) instead of NaN
        l[g] = mn == -INFINITY ? 0.f : l[g] * fast_ex2(m[g] - mn) + l2 * fast_ex2(m2 - mn);
        m[g] = mn;
      }
      if (lane == 0) m_s[warp][g] = m[g], l_s[warp][g] = l[g];
    }
  }
  __syncthreads();
  if (tid < CH_HEADS) {
    float mm = -INFINITY, L = 0.f;
#pragma unroll
    for (int w = 0; w < CH_WARPS; ++w) mm = fmaxf(mm, m_s[w][tid]);
#pragma unroll
    for (int w = 0; w < CH_WARPS; ++w)
      if (m_s[w][tid] != -INFINITY) L += l_s[w][tid] * fast_ex2(m_s[w][tid] - mm);
    lse_s[tid] = tid < H ? mm + log2f(L) : 0.f;   // key 0 always exists: L >= 1
  }
  __syncthreads();

  // ---- pass 2: p'_f of the warp's 32 keys to shared memory, then out_f += p'_f[j] v_f[j] over them
  float acc[CH_SLICES][8];
#pragma unroll
  for (int i = 0; i < CH_SLICES; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[i][e] = 0.f;
  float* pw = buf + warp * CH_HEADS * 32;
  for (int base = 32 * warp; base < nk; base += CH_THREADS) {
    const int j = base + lane;
    float pf[CH_HEADS];
#pragma unroll
    for (int f = 0; f < CH_HEADS; ++f) pf[f] = 0.f;
    if (j < nk) {
      float sm[CH_HEADS];
      scores(key_row(j), sm);
#pragma unroll
      for (int g = 0; g < CH_HEADS; ++g) {
        const float pg = fast_ex2(sm[g] - lse_s[g]);
#pragma unroll
        for (int f = 0; f < CH_HEADS; ++f) pf[f] = fmaf(lds_keep_cls(post_s + g * CH_HEADS + f), pg, pf[f]);
      }
    }
#pragma unroll
    for (int f = 0; f < CH_HEADS; ++f) pw[f * 32 + lane] = pf[f];
    __syncwarp();
    const int cnt = min(32, nk - base);
    for (int jj = 0; jj < cnt; ++jj) {
      const __nv_bfloat16* v = key_row(base + jj) + I;
#pragma unroll
      for (int i = 0; i < CH_SLICES; ++i) {
        const int c = lane + 32 * i;
        if (8 * c < I) {
          const float w = pw[(8 * c / DH) * 32 + jj];
          const uint4 raw = __ldg(reinterpret_cast<const uint4*>(v + 8 * c));
          const __nv_bfloat162* v2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 vf = __bfloat1622float2(v2[e]);
            acc[i][2 * e] = fmaf(w, vf.x, acc[i][2 * e]);
            acc[i][2 * e + 1] = fmaf(w, vf.y, acc[i][2 * e + 1]);
          }
        }
      }
    }
    __syncwarp();
  }
  __syncthreads();
  float* part = buf + warp * I;
#pragma unroll
  for (int i = 0; i < CH_SLICES; ++i) {
    const int c = lane + 32 * i;
    if (8 * c < I) {
      *reinterpret_cast<float4*>(part + 8 * c) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      *reinterpret_cast<float4*>(part + 8 * c + 4) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    }
  }
  __syncthreads();
  for (int e = 2 * tid; e < I; e += 2 * CH_THREADS) {
    float o0 = 0.f, o1 = 0.f;
#pragma unroll
    for (int w = 0; w < CH_WARPS; ++w) o0 += buf[w * I + e], o1 += buf[w * I + e + 1];
    *reinterpret_cast<__nv_bfloat162*>(p.out + (long long)b * p.ldo + e) = __floats2bfloat162_rn(o0, o1);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200vit_attention_cls_headmix(const void* qkv_self, const void* ctx_kv, int64_t ctx_ld,
                                             int64_t ctx_rows_per_image, int ctx_first, int n, void* out, int64_t ldo,
                                             int B, int H, int dh, float scale, const float* pre, const float* post,
                                             void* stream) {
  B200_CHECK_ARG(qkv_self && out && pre && post && (ctx_kv || n == 0), "attention_cls_headmix: null pointer");
  B200_CHECK_ARG(B > 0 && H > 0, "attention_cls_headmix: bad shape B=%d H=%d", B, H);
  B200_CHECK_ARG(dh == 32 || dh == 48 || dh == 64 || dh == 80 || dh == 128,
                 "attention_cls_headmix: dim_head=%d not supported (32, 48, 64, 80 or 128)", dh);
  B200_CHECK_ARG(H <= CH_HEADS, "attention_cls_headmix: H=%d > %d", H, CH_HEADS);
  B200_CHECK_ARG(H * dh <= CH_MAX_INNER, "attention_cls_headmix: H*dim_head=%d > %d", H * dh, CH_MAX_INNER);
  B200_CHECK_ARG(n >= 0 && n <= 16384, "attention_cls_headmix: n=%d context rows out of range [0, 16384]", n);
  B200_CHECK_ARG(ctx_first >= 0 && ctx_rows_per_image >= (int64_t)ctx_first + n,
                 "attention_cls_headmix: context rows [%d, %d) exceed the %lld rows per image", ctx_first,
                 ctx_first + n, (long long)ctx_rows_per_image);
  const int64_t I = (int64_t)H * dh;
  B200_CHECK_ARG(ldo >= I && (ldo % 8) == 0, "attention_cls_headmix: ldo=%lld must be >= H*dh and a multiple of 8",
                 (long long)ldo);
  B200_CHECK_ARG(n == 0 || (ctx_ld >= 2 * I && (ctx_ld % 8) == 0),
                 "attention_cls_headmix: ctx_ld=%lld must be >= 2*H*dh and a multiple of 8", (long long)ctx_ld);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv_self) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(ctx_kv) & 15) == 0,
                 "attention_cls_headmix: qkv_self, ctx_kv and out must be 16-byte aligned");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(pre) & 3) == 0 && (reinterpret_cast<uintptr_t>(post) & 3) == 0,
                 "attention_cls_headmix: pre and post must be 4-byte aligned");
  ClsHeadmixParams p{};
  p.self = reinterpret_cast<const __nv_bfloat16*>(qkv_self);
  p.ctx = reinterpret_cast<const __nv_bfloat16*>(ctx_kv);
  p.ctx_ld = ctx_ld;
  p.ctx_rows = ctx_rows_per_image;
  p.ldo = ldo;
  p.ctx_first = ctx_first;
  p.n = n;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.pre = pre;
  p.post = post;
  p.H = H;
  p.I = (int)I;
  p.scale_log2e = scale * 1.4426950408889634f;
  auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: attention_cls_headmix_kernel<32><<<B, CH_THREADS, 0, st>>>(p); break;
    case 48: attention_cls_headmix_kernel<48><<<B, CH_THREADS, 0, st>>>(p); break;
    case 80: attention_cls_headmix_kernel<80><<<B, CH_THREADS, 0, st>>>(p); break;
    case 128: attention_cls_headmix_kernel<128><<<B, CH_THREADS, 0, st>>>(p); break;
    default: attention_cls_headmix_kernel<64><<<B, CH_THREADS, 0, st>>>(p);
  }
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
