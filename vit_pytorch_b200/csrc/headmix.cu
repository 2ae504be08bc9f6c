// Attention whose heads are mixed across the head axis, for sm_90a:
//   b200vit_attention_headmix   B sequences of N tokens (1 <= N <= 16384) out of the packed q | k | v buffer
//     s_h = scale q_h k_h^T;  s'_g = sum_h pre[h][g] s_h (pre NULL: s' = s);  p_g = softmax_j(s'_g);
//     p'_f = sum_g post[g][f] p_g;  p''_f = LN over f of p' (gamma, beta, eps; head_ln NULL: p'' = p');  o_f = p''_f v_f
//   That is DeepViT's re-attention (deepvit.py:56-67: post and the LayerNorm over heads) and CaiT's talking heads
//   (cait.py:92-101: pre and post, no LayerNorm).  Every output head depends on
//   every head's probabilities at the same (i, j), so one CTA holds the score tiles of ALL heads for its query rows: no
//   score or probability tile ever goes to global memory.
//
// One CTA = 64 query rows of one sequence and 2 G output heads: two warpgroups over the same 64 rows, warpgroup w
// producing heads [y 2G + w G, y 2G + (w + 1) G).  Thread 0 loads Q (64 rows, every head) once and streams key blocks of
// 16 keys (K of every head, plus V of the CTA's 2G heads) through a two-stage TMA/mbarrier ring, twice:
//   pass 1  (warpgroup 0) S_h = Q_h K_h^T for every head (wgmma m64n16k16, operands in shared memory), pre-mixed
//           (PRE), online max / sum per (row, head) -> log2-sum-exp per (row, head) in shared memory
//   pass 2  S again (pre-mixed), p = exp2(s - lse) (exact normalised probabilities), post-mix + LayerNorm over heads in
//           fp32 registers, then O_f += P''_f V_f for the warpgroup's heads (wgmma, P'' in bf16 from registers)
// Each thread holds the same (row, key) positions of every head's tile (the wgmma accumulator layout does not depend on
// the head), so the mix is per-thread register arithmetic.  The cost of the design: every CTA computes QK^T of all H
// heads three times (pass 1 in warpgroup 0, pass 2 in both warpgroups), and a row tile has ceil(H / 2G) CTAs, so QK^T
// costs 3 ceil(H / 2G) times that of plain attention (12x at 16 x 64 and at 8 x 128 heads, 3x at 4 x 32); the mix
// costs O(H^2) fp32 FMAs per (i, j) and CTA.  G is the largest that keeps the score tiles (8 H registers) and the output accumulators
// (G dh / 2) without spills.  dh = 32, 48, 64, 80, 128 (the slab scheme of attention.cu: 64-wide 128B-swizzled and
// 16-wide 32B-swizzled slabs), H <= 16, H dh <= 1024.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int HM_ROWS = 64;
constexpr int HM_KB = 16;
constexpr int HM_THREADS = 256;
constexpr int HM_MAX_HEADS = 16;
constexpr int HM_MAX_INNER = 1024;

struct HeadmixParams {
  __nv_bfloat16* out;
  const float* post;      // [H][H]
  const float* ln_gamma;  // [H] or null (no LayerNorm over heads)
  const float* ln_beta;
  float ln_eps;
  int N, H, I;
  float scale_log2e;
  const float* pre;       // [H][H] or null (no pre-softmax mix; only the PRE instances read it)
};

// output heads per warpgroup: HC = head capacity of the instance (H <= HC).  The pre-mix needs registers of its own
// (hm_pre_span), which the 16-head instances with two or more output heads per warpgroup take from the output
// accumulators
__host__ __device__ constexpr int hm_group(int dh, int hc, bool pre = false) {
  return hc == 4 ? 2 : hc == 8 ? (dh <= 64 ? (pre && dh == 64 ? 2 : 4) : dh == 128 ? 1 : 2)
                              : (pre ? (dh <= 32 ? 2 : 1) : (dh <= 32 ? 4 : dh <= 64 ? 2 : 1));
}

// positions of a thread's 8 mixed at a time by the pre-softmax mix: HC x span temporaries
__host__ __device__ constexpr int hm_pre_span(int hc) { return hc >= 8 ? 16 / hc : 8; }

// shared memory of a CTA (offsets from the 1024B-aligned base): Q64[H][N64] | Q16[H][N16], 2 stages of
// K64[H][N64] | K16[H][N16] | V64[2G][N64] | V16[2G][N16], then lse[64][HC] | sum[64][HC], post[HC][HC] | coef[HC] |
// gamma[HC] | beta[HC] (zero-padded beyond H), pre[HC][HC] (PRE instances only), barriers full[2] empty[2] q.
// Slabs: 64-wide = rows x 128 B (128B swizzle), 16-wide = rows x 32 B (32B swizzle).
struct HmSmem {
  int q16, stage_off, k16, v64, v16, stage, lse, mix, bar, bytes;
  __host__ __device__ static int al(int x) { return (x + 1023) & ~1023; }
  __host__ __device__ HmSmem(int dh, int H, int hc, int nvh, bool pre = false) {
    const int n64 = dh / 64, n16 = (dh % 64) / 16;
    q16 = al(H * n64 * HM_ROWS * 128);
    stage_off = al(q16 + H * n16 * HM_ROWS * 32);
    k16 = al(H * n64 * HM_KB * 128);
    v64 = al(k16 + H * n16 * HM_KB * 32);
    v16 = al(v64 + nvh * n64 * HM_KB * 128);
    stage = al(v16 + nvh * n16 * HM_KB * 32);
    lse = stage_off + 2 * stage;
    mix = lse + 2 * HM_ROWS * hc * 4;  // max / log2-sum-exp and sum
    bar = mix + ((pre ? 2 : 1) * hc * hc + 3 * hc) * 4;
    bytes = bar + 5 * 8 + 1024;
  }
};

// shared-memory load the compiler may not hoist out of the key loop: the mixing weights are re-read per use instead of
// occupying H^2 registers
__device__ __forceinline__ float lds_keep(const float* p) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(smem_u32(p)));
  return v;
}
__device__ __forceinline__ float4 lds_keep4(const float* p) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(smem_u32(p)));
  return v;
}

template <int DH, int HC, bool PRE>
__global__ void __launch_bounds__(HM_THREADS, 1)
attention_headmix_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                         const __grid_constant__ CUtensorMap tmQ16, const __grid_constant__ CUtensorMap tmKV16,
                         const HeadmixParams p) {
  constexpr int N64 = DH / 64, N16 = (DH % 64) / 16, G = hm_group(DH, HC, PRE);
  static_assert(N64 * 64 + N16 * 16 == DH, "dim_head must be a multiple of 16");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int H = p.H;
  const HmSmem L(DH, H, HC, 2 * G, PRE);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L.bar);
  uint64_t* empty = full + 2;
  uint64_t* qbar = full + 4;
  float* post_s = reinterpret_cast<float*>(smem + L.mix);
  float* coef_s = post_s + HC * HC;
  float* gamma_s = coef_s + HC;
  float* beta_s = gamma_s + HC;
  float* pre_s = beta_s + HC;

  const int seq_start = blockIdx.z * p.N, len = p.N, q0 = blockIdx.x * HM_ROWS;
  const int tid = threadIdx.x;
  const int wg = tid >> 7, t = tid & 127, warp = t >> 5, lane = t & 31;
  const int hv0 = blockIdx.y * 2 * G;              // first head whose V this CTA loads
  const int nv = min(2 * G, H - hv0);
  const int f0 = hv0 + wg * G;                      // this warpgroup's first output head
  const int nf = max(0, min(G, H - f0));            // its number of output heads (0: it only keeps the ring going)
  const int nblocks = (len + HM_KB - 1) / HM_KB;
  const bool has_ln = p.ln_gamma != nullptr;
  const uint32_t kbytes = H * DH * HM_KB * 2, vbytes = nv * DH * HM_KB * 2;

  // load u of the ring: key block u of pass 1 (K), then key block u - nblocks of pass 2 (K and V)
  auto issue = [&](int u) {
    const int st = u & 1;
    const bool second = u >= nblocks;
    uint8_t* sb = smem + L.stage_off + st * L.stage;
    const int tok = (second ? u - nblocks : u) * HM_KB, z = blockIdx.z;
    mbar_arrive_expect_tx(&full[st], kbytes + (second ? vbytes : 0));
    for (int h = 0; h < H; ++h) {
#pragma unroll
      for (int c = 0; c < N64; ++c)
        tma_load_3d(sb + (h * N64 + c) * HM_KB * 128, &tmKV, &full[st], p.I + h * DH + 64 * c, tok, z);
#pragma unroll
      for (int c = 0; c < N16; ++c)
        tma_load_3d(sb + L.k16 + (h * N16 + c) * HM_KB * 32, &tmKV16, &full[st], p.I + h * DH + 64 * N64 + 16 * c,
                    tok, z);
    }
    if (second)
      for (int j = 0; j < nv; ++j) {
        const int col = 2 * p.I + (hv0 + j) * DH;
#pragma unroll
        for (int c = 0; c < N64; ++c)
          tma_load_3d(sb + L.v64 + (j * N64 + c) * HM_KB * 128, &tmKV, &full[st], col + 64 * c, tok, z);
#pragma unroll
        for (int c = 0; c < N16; ++c)
          tma_load_3d(sb + L.v16 + (j * N16 + c) * HM_KB * 32, &tmKV16, &full[st], col + 64 * N64 + 16 * c, tok, z);
      }
  };

  if (tid == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrive per warpgroup
    }
    mbar_init(qbar, 1);
    fence_mbar_init();
  }
  // mixing tables, [HC][HC] with zeros beyond H, so that the register loops run over HC heads without a branch: the
  // score tiles of heads >= H stay 0 and get weight 0.  coef[g] = mean over f of post[g][f], so that
  // mean_f p'_f = sum_g coef[g] p_g
  for (int i = tid; i < HC * HC; i += HM_THREADS) {
    const int a = i / HC, b = i % HC;
    const bool in = a < H && b < H;
    post_s[i] = in ? p.post[a * H + b] : 0.f;
    if (PRE) pre_s[i] = in ? p.pre[a * H + b] : 0.f;
  }
  for (int g = tid; g < HC; g += HM_THREADS) {
    float c = 0.f;
    for (int f = 0; g < H && f < H; ++f) c += p.post[g * H + f];
    coef_s[g] = c / H;
    gamma_s[g] = has_ln && g < H ? p.ln_gamma[g] : 1.f;
    beta_s[g] = has_ln && g < H ? p.ln_beta[g] : 0.f;
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(qbar, H * DH * HM_ROWS * 2);
    for (int h = 0; h < H; ++h) {
#pragma unroll
      for (int c = 0; c < N64; ++c)
        tma_load_3d(smem + (h * N64 + c) * HM_ROWS * 128, &tmQ, qbar, h * DH + 64 * c, q0, blockIdx.z);
#pragma unroll
      for (int c = 0; c < N16; ++c)
        tma_load_3d(smem + L.q16 + (h * N16 + c) * HM_ROWS * 32, &tmQ16, qbar, h * DH + 64 * N64 + 16 * c, q0,
                    blockIdx.z);
    }
    issue(0);
    issue(1);  // 2 nblocks >= 2 loads
  }

  const uint32_t qa = smem_u32(smem), qa16 = smem_u32(smem + L.q16);
  // s[h][4 j + 2 r + c]: row 16 warp + lane / 4 + 8 r, key 8 j + 2 (lane % 4) + c of the block
  float s[HC][8];
#pragma unroll
  for (int h = 0; h < HC; ++h)
#pragma unroll
    for (int e = 0; e < 8; ++e) s[h][e] = 0.f;

  // S_h = Q_h K_h^T of every head, scaled, in log2 units
  auto scores = [&](uint32_t sb) {
    wgmma_fence();
#pragma unroll
    for (int h = 0; h < HC; ++h) {
      // heads beyond H issue no MMA.  H is a run-time value, so ptxas treats this warp-uniform branch as divergent and
      // inserts a warpgroup.arrive before the MMAs (C7519); issuing them unconditionally on a clamped head index
      // instead costs registers and made three instances spill
      if (h < H) {
#pragma unroll
        for (int c = 0; c < N64; ++c)
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint64_t ad = make_wgmma_desc(qa + (h * N64 + c) * HM_ROWS * 128, 1024, WGMMA_SW128) + 2 * k;
            const uint64_t bd = make_wgmma_desc(sb + (h * N64 + c) * HM_KB * 128, 1024, WGMMA_SW128) + 2 * k;
            wgmma_m64n16k16(s[h], ad, bd, c != 0 || k != 0);
          }
#pragma unroll
        for (int c = 0; c < N16; ++c) {
          const uint64_t ad = make_wgmma_desc(qa16 + (h * N16 + c) * HM_ROWS * 32, 256, WGMMA_SW32);
          const uint64_t bd = make_wgmma_desc(sb + L.k16 + (h * N16 + c) * HM_KB * 32, 256, WGMMA_SW32);
          wgmma_m64n16k16(s[h], ad, bd, N64 != 0 || c != 0);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < HC; ++h) fence_regs(s[h]);
    // heads >= H have no MMA: a 0 tile (a masked -inf left from an earlier block times a 0 weight would be NaN)
#pragma unroll
    for (int h = 0; h < HC; ++h)
#pragma unroll
      for (int e = 0; e < 8; ++e) s[h][e] = h < H ? s[h][e] : 0.f;
#pragma unroll
    for (int h = 0; h < HC; ++h)
#pragma unroll
      for (int e = 0; e < 8; ++e) s[h][e] *= p.scale_log2e;
    if constexpr (PRE) {
      // s'_g = sum_h pre[h][g] s_h, in place, SP positions at a time.  Linear, so it commutes with scale_log2e; it
      // runs before the key mask (a masked -inf inside the sum would give NaN), heads >= H are 0 with weight 0.  A
      // rolled loop: each step mixes positions 0..SP-1 and rotates the 8 positions left by SP (register moves), so
      // that ptxas cannot overlap the steps, whose temporaries together would not fit next to the score tiles
      constexpr int SP = hm_pre_span(HC), e0 = 0;
#pragma unroll 1
      for (int step = 0; step < 8 / SP; ++step) {
        float m[HC][SP];
#pragma unroll
        for (int g = 0; g < HC; ++g)
#pragma unroll
          for (int e = 0; e < SP; ++e) m[g][e] = 0.f;
#pragma unroll
        for (int h = 0; h < HC; ++h)
#pragma unroll
          for (int g = 0; g < HC; g += 4) {
            const float4 w = lds_keep4(pre_s + h * HC + g);   // pre_s is 16-byte aligned (L.mix + post + 3 HC)
#pragma unroll
            for (int e = 0; e < SP; ++e) {
              m[g][e] = fmaf(w.x, s[h][e0 + e], m[g][e]);
              m[g + 1][e] = fmaf(w.y, s[h][e0 + e], m[g + 1][e]);
              m[g + 2][e] = fmaf(w.z, s[h][e0 + e], m[g + 2][e]);
              m[g + 3][e] = fmaf(w.w, s[h][e0 + e], m[g + 3][e]);
            }
          }
#pragma unroll
        for (int g = 0; g < HC; ++g) {
#pragma unroll
          for (int e = 0; e + SP < 8; ++e) s[g][e] = s[g][e + SP];
#pragma unroll
          for (int e = 0; e < SP; ++e) s[g][8 - SP + e] = m[g][e];
        }
      }
    }
  };
  auto key_ok = [&](int kb, int e) { return kb * HM_KB + 8 * (e >> 2) + 2 * (lane & 3) + (e & 1) < len; };
  auto release = [&](int u) {
    if (t == 0) mbar_arrive(&empty[u & 1]);
    if (tid == 0 && u + 2 < 2 * nblocks) {
      mbar_wait(&empty[u & 1], (u >> 1) & 1);  // both warpgroups are done with this stage
      issue(u + 2);
    }
  };

  mbar_wait(qbar, 0);
  // [64][HC] running max, then log2-sum-exp, and [64][HC] running sum, of warpgroup 0's pass 1 (the entries of a row
  // belong to the thread of its quad with lane % 4 == 0)
  float* lse_s = reinterpret_cast<float*>(smem + L.lse);
  float* sum_s = lse_s + HM_ROWS * HC;
  const int lrow = 16 * warp + (lane >> 2);

  // ---- pass 1 (warpgroup 0; warpgroup 1 only releases the stages): per (row, mixed head) max and sum of exp2 over
  // all keys.  Per block: the quad's block max bm and sum of exp2(s - bm), merged into the running pair in shared
  // memory, which keeps the registers to the score tiles.
  for (int kb = 0; kb < nblocks; ++kb) {
    const int st = kb & 1;
    mbar_wait(&full[st], (kb >> 1) & 1);
    if (wg == 0) {
      scores(smem_u32(smem + L.stage_off + st * L.stage));
#pragma unroll
      for (int g = 0; g < HC; ++g) {
#pragma unroll
        for (int e = 0; e < 8; ++e) s[g][e] = key_ok(kb, e) ? s[g][e] : -INFINITY;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float bm = fmaxf(fmaxf(s[g][2 * r], s[g][2 * r + 1]), fmaxf(s[g][4 + 2 * r], s[g][5 + 2 * r]));
          bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 1));
          bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 2));
          // a block whose keys are all beyond the sequence (none: every block holds key kb * 16 < len) would give
          // bm = -inf; key kb * 16 is valid, so bm is finite
          float bs = fast_ex2(s[g][2 * r] - bm) + fast_ex2(s[g][2 * r + 1] - bm) + fast_ex2(s[g][4 + 2 * r] - bm) +
                     fast_ex2(s[g][5 + 2 * r] - bm);
          bs += __shfl_xor_sync(0xffffffffu, bs, 1);
          bs += __shfl_xor_sync(0xffffffffu, bs, 2);
          if ((lane & 3) == 0) {
            const int i = (lrow + 8 * r) * HC + g;
            if (kb == 0) {
              lse_s[i] = bm;
              sum_s[i] = bs;
            } else {
              const float m0 = lse_s[i], mx = fmaxf(m0, bm);
              sum_s[i] = sum_s[i] * fast_ex2(m0 - mx) + bs * fast_ex2(bm - mx);
              lse_s[i] = mx;
            }
          }
        }
      }
    }
    release(kb);
  }
  if (wg == 0 && (lane & 3) == 0) {
#pragma unroll
    for (int g = 0; g < HC; ++g)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int i = (lrow + 8 * r) * HC + g;
        lse_s[i] += __log2f(sum_s[i]);
      }
  }
  __syncthreads();

  // ---- pass 2: probabilities, post-mix, LayerNorm over heads, O += P'' V
  float o[G][N64 > 0 ? N64 : 1][32], o16[G][N16 > 0 ? N16 : 1][8];
#pragma unroll
  for (int gi = 0; gi < G; ++gi) {
#pragma unroll
    for (int c = 0; c < N64; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[gi][c][i] = 0.f;
#pragma unroll
    for (int c = 0; c < N16; ++c)
#pragma unroll
      for (int i = 0; i < 8; ++i) o16[gi][c][i] = 0.f;
  }
  for (int kb = 0; kb < nblocks; ++kb) {
    const int u = nblocks + kb, st = u & 1;
    mbar_wait(&full[st], (u >> 1) & 1);
    const uint32_t sb = smem_u32(smem + L.stage_off + st * L.stage);
    if (nf > 0) {
      scores(sb);
#pragma unroll
      for (int g = 0; g < HC; ++g) {
        const float lse0 = lds_keep(lse_s + lrow * HC + g), lse1 = lds_keep(lse_s + (lrow + 8) * HC + g);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          s[g][e] = key_ok(kb, e) ? fast_ex2(s[g][e] - ((e & 2) ? lse1 : lse0)) : 0.f;
      }
      // LayerNorm statistics over the H post-mixed heads of each position
      float mean[8], rstd[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) mean[e] = 0.f, rstd[e] = 0.f;
      if (has_ln) {
#pragma unroll
        for (int g = 0; g < HC; ++g) {
          const float c = lds_keep(coef_s + g);
#pragma unroll
          for (int e = 0; e < 8; ++e) mean[e] = fmaf(c, s[g][e], mean[e]);
        }
        for (int f = 0; f < H; ++f) {
          float acc[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
          for (int g = 0; g < HC; ++g) {
            const float w = lds_keep(post_s + g * HC + f);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = fmaf(w, s[g][e], acc[e]);
          }
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const float d = acc[e] - mean[e];
            rstd[e] = fmaf(d, d, rstd[e]);
          }
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) rstd[e] = rsqrtf(rstd[e] / H + p.ln_eps);
      }
      // P''_f of the warpgroup's heads as bf16 A fragments; keys beyond the sequence get 0 (after the LayerNorm,
      // which would give them beta)
      uint32_t a[G][4];
#pragma unroll
      for (int gi = 0; gi < G; ++gi) {
        const int f = f0 + gi;
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
        if (gi < nf) {
#pragma unroll
          for (int g = 0; g < HC; ++g) {
            const float w = lds_keep(post_s + g * HC + f);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = fmaf(w, s[g][e], acc[e]);
          }
          if (has_ln) {
            const float ga = lds_keep(gamma_s + f), be = lds_keep(beta_s + f);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = fmaf((acc[e] - mean[e]) * rstd[e], ga, be);
          }
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] = key_ok(kb, e) ? acc[e] : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) a[gi][i] = pack_bf16x2(acc[2 * i], acc[2 * i + 1]);
      }
      wgmma_fence();
#pragma unroll
      for (int gi = 0; gi < G; ++gi) {
        if (gi >= nf) continue;
        const int j = wg * G + gi;  // V slot of the head in the stage
#pragma unroll
        for (int c = 0; c < N64; ++c)
          wgmma_m64n64k16_rs_tb(o[gi][c], a[gi],
                                make_wgmma_desc_lbo(sb + L.v64 + (j * N64 + c) * HM_KB * 128, 1024, 1024, WGMMA_SW128));
#pragma unroll
        for (int c = 0; c < N16; ++c)
          wgmma_m64n16k16_rs_tb(o16[gi][c], a[gi],
                                make_wgmma_desc_lbo(sb + L.v16 + (j * N16 + c) * HM_KB * 32, 256, 256, WGMMA_SW32));
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int gi = 0; gi < G; ++gi) {
#pragma unroll
        for (int c = 0; c < N64; ++c) fence_regs(o[gi][c]);
#pragma unroll
        for (int c = 0; c < N16; ++c) fence_regs(o16[gi][c]);
      }
    }
    release(u);
  }

  const int qr = q0 + lrow;
#pragma unroll
  for (int gi = 0; gi < G; ++gi) {
    if (gi >= nf) continue;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = qr + 8 * r;
      if (row >= len) continue;
      __nv_bfloat16* op = p.out + (long long)(seq_start + row) * p.I + (f0 + gi) * DH + 2 * (lane & 3);
#pragma unroll
      for (int c = 0; c < N64; ++c)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint32_t*>(op + 64 * c + j * 8) =
              pack_bf16x2(o[gi][c][4 * j + 2 * r], o[gi][c][4 * j + 2 * r + 1]);
#pragma unroll
      for (int c = 0; c < N16; ++c)
#pragma unroll
        for (int j = 0; j < 2; ++j)
          *reinterpret_cast<uint32_t*>(op + 64 * N64 + 16 * c + j * 8) =
              pack_bf16x2(o16[gi][c][4 * j + 2 * r], o16[gi][c][4 * j + 2 * r + 1]);
    }
  }
}

template <int DH, int HC, bool PRE>
static int launch_headmix_t(const void* qkv, int B, const HeadmixParams& p, cudaStream_t stream) {
  constexpr int G = hm_group(DH, HC, PRE);
  const HmSmem L(DH, p.H, HC, 2 * G, PRE);
  B200_CHECK_ARG(L.bytes <= 227 * 1024, "attention_headmix: H=%d dh=%d needs %d bytes of shared memory", p.H, DH,
                 L.bytes);
  // the [B][N][3 I] view (column, token, sequence): boxes past the end of a sequence are zero-filled, so that a
  // sequence never reads another's rows (0 x NaN in O += P'' V would be NaN)
  CUtensorMap tm[4];
  const uint64_t ld = (uint64_t)3 * p.I;
  const uint64_t dims[3] = {ld, (uint64_t)p.N, (uint64_t)B};
  const uint64_t strides[2] = {ld * 2, ld * 2 * p.N};
  const uint32_t qbox[3] = {64, HM_ROWS, 1}, kvbox[3] = {64, HM_KB, 1}, qbox16[3] = {16, HM_ROWS, 1},
                 kvbox16[3] = {16, HM_KB, 1};
  constexpr bool has64 = DH / 64 > 0, has16 = (DH % 64) / 16 > 0;
  int rc = 0;
  if (has64) rc = encode_tmap_bf16(&tm[0], qkv, 3, dims, strides, qbox);
  if (!rc && has64) rc = encode_tmap_bf16(&tm[1], qkv, 3, dims, strides, kvbox);
  if (!rc && has16) rc = encode_tmap_bf16_sw(&tm[2], qkv, 3, dims, strides, qbox16, 32);
  if (!rc && has16) rc = encode_tmap_bf16_sw(&tm[3], qkv, 3, dims, strides, kvbox16, 32);
  if (rc) return rc;
  if (!has16) tm[2] = tm[0], tm[3] = tm[1];
  if (!has64) tm[0] = tm[2], tm[1] = tm[3];
  auto kern = attention_headmix_kernel<DH, HC, PRE>;
  B200_ENSURE_SMEM(kern, L.bytes);
  const dim3 grid((p.N + HM_ROWS - 1) / HM_ROWS, (p.H + 2 * G - 1) / (2 * G), B);
  kern<<<grid, HM_THREADS, L.bytes, stream>>>(tm[0], tm[1], tm[2], tm[3], p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

template <int DH, bool PRE>
static int launch_headmix_hc(const void* qkv, int B, const HeadmixParams& p, cudaStream_t st) {
  if (p.H <= 4) return launch_headmix_t<DH, 4, PRE>(qkv, B, p, st);
  if constexpr (DH == 128) return launch_headmix_t<DH, 8, PRE>(qkv, B, p, st);  // H dh <= 1024: H <= 8
  else return p.H <= 8 ? launch_headmix_t<DH, 8, PRE>(qkv, B, p, st) : launch_headmix_t<DH, 16, PRE>(qkv, B, p, st);
}

template <int DH>
static int launch_headmix_dh(const void* qkv, int B, const HeadmixParams& p, cudaStream_t st) {
  return p.pre ? launch_headmix_hc<DH, true>(qkv, B, p, st) : launch_headmix_hc<DH, false>(qkv, B, p, st);
}

}  // namespace b200

using namespace b200;

extern "C" int b200vit_attention_headmix_ex(const void* qkv, void* out, int B, int N, int H, int dh, float scale,
                                            const float* pre, const float* post, const float* head_ln_gamma,
                                            const float* head_ln_beta, float head_ln_eps, void* stream) {
  B200_CHECK_ARG(qkv && out && post, "attention_headmix: null pointer");
  B200_CHECK_ARG((head_ln_gamma == nullptr) == (head_ln_beta == nullptr),
                 "attention_headmix: head LayerNorm needs both gamma and beta");
  B200_CHECK_ARG(B > 0 && N > 0 && H > 0, "attention_headmix: bad shape B=%d N=%d H=%d", B, N, H);
  B200_CHECK_ARG(dh == 32 || dh == 48 || dh == 64 || dh == 80 || dh == 128,
                 "attention_headmix: dim_head=%d not supported (32, 48, 64, 80 or 128)", dh);
  B200_CHECK_ARG(H <= HM_MAX_HEADS, "attention_headmix: H=%d > %d", H, HM_MAX_HEADS);
  B200_CHECK_ARG(H * dh <= HM_MAX_INNER, "attention_headmix: H*dim_head=%d > %d", H * dh, HM_MAX_INNER);
  B200_CHECK_ARG(N <= 16384, "attention_headmix: N=%d > 16384", N);
  B200_CHECK_ARG(B <= 65535, "attention_headmix: B=%d exceeds the grid", B);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "attention_headmix: qkv and out must be 16-byte aligned");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(post) & 3) == 0 && (reinterpret_cast<uintptr_t>(pre) & 3) == 0 &&
                     (reinterpret_cast<uintptr_t>(head_ln_gamma) & 3) == 0 &&
                     (reinterpret_cast<uintptr_t>(head_ln_beta) & 3) == 0,
                 "attention_headmix: pre, post and head LayerNorm vectors must be 4-byte aligned");
  B200_CHECK_ARG(head_ln_gamma == nullptr || head_ln_eps > 0.f, "attention_headmix: head LayerNorm eps must be > 0");
  HeadmixParams p{};
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.post = post;
  p.pre = pre;
  p.ln_gamma = head_ln_gamma;
  p.ln_beta = head_ln_beta;
  p.ln_eps = head_ln_eps;
  p.N = N;
  p.H = H;
  p.I = H * dh;
  p.scale_log2e = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: return launch_headmix_dh<32>(qkv, B, p, st);
    case 48: return launch_headmix_dh<48>(qkv, B, p, st);
    case 80: return launch_headmix_dh<80>(qkv, B, p, st);
    case 128: return launch_headmix_dh<128>(qkv, B, p, st);
    default: return launch_headmix_dh<64>(qkv, B, p, st);
  }
}

extern "C" int b200vit_attention_headmix(const void* qkv, void* out, int B, int N, int H, int dh, float scale,
                                         const float* post, const float* head_ln_gamma,
                                         const float* head_ln_beta, float head_ln_eps, void* stream) {
  return b200vit_attention_headmix_ex(qkv, out, B, N, H, dh, scale, nullptr, post, head_ln_gamma, head_ln_beta,
                                      head_ln_eps, stream);
}
