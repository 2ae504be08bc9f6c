// Kernels of the hierarchical, window-attention models (Twins-SVT, reference twins_svt.py), for sm_90a.  The token map
// of a stage is kept token-major: x[B*gh*gw, C], token (b, y, x) at row (b*gh + y)*gw + x.  The window attention,
// b200vit_attention_window, is in attention_tile64.cu.
//   b200vit_attention_kv       every query of an image against that image's keys / values, which come from another
//                              buffer and have another length (twins_svt.py:122-157: the sub-sampled keys);
//                              b200vit_attention_kv_ex takes key heads of another width than the value heads
//                              (ScalableViT's SSA, scalable_vit.py:71-124); b200vit_attention_kv_lens takes each
//                              image's key count from a device array (Adaptive Token Sampling, ats_vit.py)
//   b200vit_merge_patches_ln   p x p patch merging + LayerNorm over the merged features (twins_svt.py:59-75)
//   b200vit_peg                depthwise k x k convolution plus identity (twins_svt.py:77-83)
//
// attention_kv: one CTA = two warpgroups = one (image, head) and a strided share of its 128-row query tiles, 64 rows
// per warpgroup.  Keys and values are cut in blocks of 64 that thread 0 loads with TMA over the 3-D view (column, key,
// image) of kv, keys past Nk zero-filled.  Most of the work of a CTA is on the query side (Nq >> Nk in Twins-SVT: 3136
// queries against 64 keys), so when all key blocks of the (image, head) fit the CTA's shared memory they are loaded
// once and every query tile of the CTA loops over them; otherwise they stream through a ring of 4 block slots, loaded
// 3 blocks ahead, once per query tile.  Per block: S = Q K^T with wgmma, keys past Nk masked to -inf, the online
// softmax of attention.cu in fp32, O += P V with wgmma (P from registers, V as the transposed B operand).  The
// resident / streaming choice and the CTA count are untuned: no measurement preceded them.
#include "tile64.cuh"
#include "host_util.h"

namespace b200 {

using namespace tile64;

// ------------------------------------------------------------------------------------------------ attention_kv
constexpr int KV_THREADS = 256;
constexpr int KV_RING = 4;             // block slots of the streaming mode
constexpr int KV_SMEM = 200 * 1024;    // what a CTA may hold: the query tile and the resident key / value blocks
constexpr int KV_MAX_SLOTS = 16;

template <int DK, int DV>
constexpr int kv_resident_slots() {
  const int n = (KV_SMEM - 2 * Slabs<DK>::OP) / (Slabs<DK>::OP + Slabs<DV>::OP);
  return n < KV_MAX_SLOTS ? n : KV_MAX_SLOTS;
}

struct KvParams {
  __nv_bfloat16* out;
  int B, Nq, Nk;
  int Ik, Iv;              // H * dk (q and k columns), H * dv (v and out columns)
  int slots;               // block slots in shared memory; all blocks resident iff ceil(Nk / 64) <= slots
  float scale_log2e;
  const int* nk;           // LENS: keys of image b = nk[b], clamped to [1, Nk] (b200vit_attention_kv_lens)
};

// DK: width of the q and k heads, DV: of the v and output heads; LENS: per-image key counts from p.nk
template <int DK, int DV, bool LENS = false>
__global__ void __launch_bounds__(KV_THREADS)
attention_kv_kernel(const __grid_constant__ CUtensorMap q64, const __grid_constant__ CUtensorMap q16,
                    const __grid_constant__ CUtensorMap kv64, const __grid_constant__ CUtensorMap kv16,
                    const KvParams p) {
  using S = Slabs<DK>;
  using SV = Slabs<DV>;
  constexpr int N64 = SV::N64, N16 = SV::N16;
  constexpr int SLOT = S::OP + SV::OP;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // Q: two operand blocks (one per warpgroup); then per slot K | V; then the barriers: Q, one per slot
  uint8_t* slot0 = smem + 2 * S::OP;
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(slot0 + (size_t)p.slots * SLOT);
  uint64_t* bar_kv = bar_q + 1;

  const int h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  const int Nk = LENS ? min(max(p.nk[b], 1), p.Nk) : p.Nk;
  const int nqt = (p.Nq + 127) / 128, nkb = (Nk + 63) / 64;
  const bool resident = nkb <= p.slots;

  if (tid == 0) {
    tma_prefetch_desc(S::N64 ? &q64 : &q16);
    tma_prefetch_desc(S::N64 ? &kv64 : &kv16);
    mbar_init(bar_q, 1);
    for (int i = 0; i < p.slots; ++i) mbar_init(bar_kv + i, 1);
    fence_mbar_init();
  }

  auto load_block = [&](int j) {  // thread 0: keys [64 j, 64 j + 64) of image b into slot j % slots
    const int sl = j % p.slots;
    uint8_t* dst = slot0 + (size_t)sl * SLOT;
    mbar_arrive_expect_tx(bar_kv + sl, ROWS * (DK + DV) * 2);
    const int ck = h * DK;
#pragma unroll
    for (int c = 0; c < S::N64; ++c) tma_load_3d(dst + c * S::S64, &kv64, bar_kv + sl, ck + 64 * c, 64 * j, b);
#pragma unroll
    for (int c = 0; c < S::N16; ++c)
      tma_load_3d(dst + S::N64 * S::S64 + c * S::S16, &kv16, bar_kv + sl, ck + 64 * S::N64 + 16 * c, 64 * j, b);
    const int cv = p.Ik + h * DV;
#pragma unroll
    for (int c = 0; c < N64; ++c) tma_load_3d(dst + S::OP + c * SV::S64, &kv64, bar_kv + sl, cv + 64 * c, 64 * j, b);
#pragma unroll
    for (int c = 0; c < N16; ++c)
      tma_load_3d(dst + S::OP + N64 * SV::S64 + c * SV::S16, &kv16, bar_kv + sl, cv + 64 * N64 + 16 * c, 64 * j, b);
  };

  uint32_t q_phase = 0, kv_phase = 0;  // kv_phase: one bit per slot
  bool first = true;
  for (int qt = blockIdx.x; qt < nqt; qt += gridDim.x, first = false) {
    const int q0 = qt * 128;
    __syncthreads();  // the barriers are initialised; every thread is done with the previous tile's Q (and slots)
    if (tid == 0) {
      mbar_arrive_expect_tx(bar_q, 2 * ROWS * DK * 2);
#pragma unroll
      for (int w = 0; w < 2; ++w) {
#pragma unroll
        for (int c = 0; c < S::N64; ++c)
          tma_load_3d(smem + w * S::OP + c * S::S64, &q64, bar_q, h * DK + 64 * c, q0 + 64 * w, b);
#pragma unroll
        for (int c = 0; c < S::N16; ++c)
          tma_load_3d(smem + w * S::OP + S::N64 * S::S64 + c * S::S16, &q16, bar_q, h * DK + 64 * S::N64 + 16 * c,
                      q0 + 64 * w, b);
      }
      if (resident) {
        if (first)
          for (int j = 0; j < nkb; ++j) load_block(j);
      } else {
        for (int j = 0; j < p.slots - 1 && j < nkb; ++j) load_block(j);
      }
    }

    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[N64 > 0 ? N64 : 1][32], o16[N16 > 0 ? N16 : 1][8];
#pragma unroll
    for (int c = 0; c < N64; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
#pragma unroll
    for (int c = 0; c < N16; ++c)
#pragma unroll
      for (int i = 0; i < 8; ++i) o16[c][i] = 0.f;

    mbar_wait(bar_q, q_phase);
    q_phase ^= 1;
    const uint32_t sq = smem_u32(smem) + wg * S::OP;

    for (int kb = 0; kb < nkb; ++kb) {
      const int sl = kb % p.slots;
      if (!resident) {
        __syncthreads();  // every thread is done with block kb - 1: its slot takes block kb + slots - 1
        if (tid == 0 && kb + p.slots - 1 < nkb) load_block(kb + p.slots - 1);
      }
      if (first || !resident) {
        mbar_wait(bar_kv + sl, (kv_phase >> sl) & 1u);
        kv_phase ^= 1u << sl;
      }
      const uint32_t sk = smem_u32(slot0) + sl * SLOT, sv = sk + S::OP;

      float s[32];
      wgmma_fence();
      qk_mma<DK>(s, sq, sk);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);

      // online softmax in log2 units; s[4 jj + e]: row half e >> 1, key 64 kb + 8 jj + 2 (lane % 4) + (e & 1)
      const int key0 = 64 * kb + 2 * (lane & 3);
      float mn[2] = {m[0], m[1]};
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int rh = e >> 1;
          s[4 * jj + e] = key0 + 8 * jj + (e & 1) < Nk ? s[4 * jj + e] * p.scale_log2e : -INFINITY;
          mn[rh] = fmaxf(mn[rh], s[4 * jj + e]);
        }
      float alpha[2];
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        mn[rh] = fmaxf(mn[rh], __shfl_xor_sync(0xffffffffu, mn[rh], 1));
        mn[rh] = fmaxf(mn[rh], __shfl_xor_sync(0xffffffffu, mn[rh], 2));
        // every block holds at least one key, so mn is finite unless the scores are not
        alpha[rh] = fast_ex2(m[rh] - mn[rh]);
        m[rh] = mn[rh];
        l[rh] *= alpha[rh];
      }
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int rh = e >> 1;
          const float v = fast_ex2(s[4 * jj + e] - m[rh]);
          s[4 * jj + e] = v;
          l[rh] += v;  // this thread's keys only: summed over the four lanes of the row after the last block
        }
#pragma unroll
      for (int c = 0; c < N64; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[c][i] *= alpha[(i >> 1) & 1];
#pragma unroll
      for (int c = 0; c < N16; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) o16[c][i] *= alpha[(i >> 1) & 1];
#pragma unroll
      for (int c = 0; c < N64; ++c) fence_regs(o[c]);
#pragma unroll
      for (int c = 0; c < N16; ++c) fence_regs(o16[c]);
      wgmma_fence();
      pv_mma<DV>(o, o16, s, sv);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < N64; ++c) fence_regs(o[c]);
#pragma unroll
      for (int c = 0; c < N16; ++c) fence_regs(o16[c]);
    }

#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 1);
      l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 2);
      const int q = q0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * rh;
      if (q >= p.Nq) continue;
      store_rows<DV>(o, o16, p.out + ((long long)b * p.Nq + q) * p.Iv + h * DV + 2 * (lane & 3), rh, 1.0f / l[rh]);
    }
  }
}

template <int DK, int DV, bool LENS = false>
static int launch_kv_t(const void* q, int64_t ldq, const void* kv, int64_t ldkv, KvParams p, int H,
                       cudaStream_t stream) {
  using S = Slabs<DK>;
  using SV = Slabs<DV>;
  CUtensorMap tm[4];
  const uint64_t qdims[3] = {(uint64_t)p.Ik, (uint64_t)p.Nq, (uint64_t)p.B};
  const uint64_t qstr[2] = {(uint64_t)ldq * 2, (uint64_t)ldq * 2 * p.Nq};
  const uint64_t kdims[3] = {(uint64_t)(p.Ik + p.Iv), (uint64_t)p.Nk, (uint64_t)p.B};
  const uint64_t kstr[2] = {(uint64_t)ldkv * 2, (uint64_t)ldkv * 2 * p.Nk};
  const uint32_t box64[3] = {64, ROWS, 1}, box16[3] = {16, ROWS, 1};
  // q64 / q16 serve the q blocks; kv64 / kv16 the k and v blocks, whichever slab widths the two have
  constexpr bool q64 = S::N64 > 0, q16 = S::N16 > 0, kv64 = S::N64 + SV::N64 > 0, kv16 = S::N16 + SV::N16 > 0;
  int rc = 0;
  if (q64) rc = encode_tmap_bf16(&tm[0], q, 3, qdims, qstr, box64);
  if (!rc && kv64) rc = encode_tmap_bf16(&tm[2], kv, 3, kdims, kstr, box64);
  if (!rc && q16) rc = encode_tmap_bf16_sw(&tm[1], q, 3, qdims, qstr, box16, 32);
  if (!rc && kv16) rc = encode_tmap_bf16_sw(&tm[3], kv, 3, kdims, kstr, box16, 32);
  if (rc) return rc;
  if (!q16) tm[1] = tm[0];
  if (!q64) tm[0] = tm[1];
  if (!kv16) tm[3] = tm[2];
  if (!kv64) tm[2] = tm[3];
  const int nkb = (p.Nk + 63) / 64, nqt = (p.Nq + 127) / 128;
  p.slots = nkb <= kv_resident_slots<DK, DV>() ? nkb : KV_RING;
  const int bytes = 2 * S::OP + p.slots * (S::OP + SV::OP) + 8 * (1 + KV_MAX_SLOTS) + 1024;
  // enough CTAs to fill the device about twice; an (image, head) with resident keys is not split further than that
  const long long pairs = (long long)p.B * H;
  long long per = (2LL * num_sms() + pairs - 1) / pairs;
  if (per > nqt) per = nqt;
  if (per < 1) per = 1;
  auto kern = attention_kv_kernel<DK, DV, LENS>;
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3((unsigned)per, H, p.B), KV_THREADS, bytes, stream>>>(tm[0], tm[1], tm[2], tm[3], p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------ merge_patches_ln
// One warp per output row: the p*p tokens of the block, C contiguous floats each, are read three times (mean, variance,
// output) out of L1 / L2.
__global__ void __launch_bounds__(256)
merge_patches_ln_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                        __nv_bfloat16* __restrict__ out, long long ldo, int rows, int gh, int gw, int C, int p,
                        float eps) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int oh = gh / p, ow = gw / p;
  const int b = row / (oh * ow), oy = (row / ow) % oh, ox = row % ow;
  const float* base = x + (((long long)b * gh + oy * p) * gw + ox * p) * C;
  const int C4 = C >> 2, K4 = p * p * C4;
  auto src = [&](int i) {  // float4 index i of the merged row: tap i / C4 = p1 * p + p2
    const int t = i / C4, c4 = i - t * C4;
    return reinterpret_cast<const float4*>(base + ((long long)(t / p) * gw + t % p) * C) + c4;
  };
  float s = 0.f;
  for (int i = lane; i < K4; i += 32) {
    const float4 v = *src(i);
    s += (v.x + v.y) + (v.z + v.w);
  }
  const float mean = warp_sum(s) / (float)(4 * K4);
  float q = 0.f;
  for (int i = lane; i < K4; i += 32) {
    const float4 v = *src(i);
    const float a = v.x - mean, bb = v.y - mean, c = v.z - mean, d = v.w - mean;
    q += (a * a + bb * bb) + (c * c + d * d);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)(4 * K4) + eps);
  __nv_bfloat16* orow = out + (long long)row * ldo;
  for (int i = lane; i < K4; i += 32) {
    const float4 v = *src(i);
    const float4 g = *reinterpret_cast<const float4*>(gamma + 4 * i);
    const float4 bt = *reinterpret_cast<const float4*>(beta + 4 * i);
    uint2 pk;
    pk.x = pack_bf16x2((v.x - mean) * rstd * g.x + bt.x, (v.y - mean) * rstd * g.y + bt.y);
    pk.y = pack_bf16x2((v.z - mean) * rstd * g.z + bt.z, (v.w - mean) * rstd * g.w + bt.w);
    *reinterpret_cast<uint2*>(orow + 4 * i) = pk;
  }
  for (long long i = 4LL * K4 + lane; i < ldo; i += 32) orow[i] = __float2bfloat16_rn(0.f);
}

// ------------------------------------------------------------------------------------------------ peg
// One thread per token and 4 channels; the k x k neighbourhood comes out of L1 / L2.
__global__ void __launch_bounds__(256)
peg_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
           float* __restrict__ y, long long total4, int gh, int gw, int C, int k) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= total4) return;
  const int C4 = C >> 2;
  const int c = (int)(i % C4) * 4;
  const long long tok = i / C4;
  const int xx = (int)(tok % gw), yy = (int)((tok / gw) % gh);
  const int r = k >> 1;
  float4 acc = *reinterpret_cast<const float4*>(bias + c);
  for (int dy = 0; dy < k; ++dy) {
    const int sy = yy + dy - r;
    if (sy < 0 || sy >= gh) continue;
    for (int dx = 0; dx < k; ++dx) {
      const int sx = xx + dx - r;
      if (sx < 0 || sx >= gw) continue;
      const float4 v = *reinterpret_cast<const float4*>(x + (tok + (long long)(dy - r) * gw + (dx - r)) * C + c);
      const float4 ww = *reinterpret_cast<const float4*>(w + (long long)(dy * k + dx) * C + c);
      acc.x = fmaf(ww.x, v.x, acc.x);
      acc.y = fmaf(ww.y, v.y, acc.y);
      acc.z = fmaf(ww.z, v.z, acc.z);
      acc.w = fmaf(ww.w, v.w, acc.w);
    }
  }
  const float4 v = *reinterpret_cast<const float4*>(x + tok * C + c);
  *reinterpret_cast<float4*>(y + tok * C + c) = make_float4(acc.x + v.x, acc.y + v.y, acc.z + v.z, acc.w + v.w);
}

}  // namespace b200

using namespace b200;

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static bool overlap(const void* a, long long a_bytes, const void* b, long long b_bytes) {
  const uintptr_t p = reinterpret_cast<uintptr_t>(a), q = reinterpret_cast<uintptr_t>(b);
  return p < q + (uintptr_t)b_bytes && q < p + (uintptr_t)a_bytes;
}

// the checks and launch shared by b200vit_attention_kv (dk == dv) and b200vit_attention_kv_ex; `what` names the caller
// (check_overlap: out must overlap neither q nor kv, which b200vit_attention_kv has never checked)
static int attention_kv_impl(const char* what, const void* q, int64_t ldq, const void* kv, int64_t ldkv, void* out,
                             int B, int Nq, int Nk, int H, int dk, int dv, float scale, void* stream,
                             bool check_overlap = false) {
  B200_CHECK_ARG(q && kv && out, "%s: null pointer", what);
  B200_CHECK_ARG(B > 0 && Nq > 0 && Nk > 0 && H > 0, "%s: bad shape B=%d Nq=%d Nk=%d H=%d", what, B, Nq, Nk, H);
  B200_CHECK_ARG(Nk <= B200VIT_ATTN_KV_MAX_KEYS, "%s: Nk=%d > %d", what, Nk, B200VIT_ATTN_KV_MAX_KEYS);
  B200_CHECK_ARG(ldq >= (int64_t)H * dk && ldq % 8 == 0, "%s: ldq=%lld must be a multiple of 8 and >= %d", what,
                 (long long)ldq, H * dk);
  B200_CHECK_ARG(ldkv >= (int64_t)H * (dk + dv) && ldkv % 8 == 0, "%s: ldkv=%lld must be a multiple of 8 and >= %d",
                 what, (long long)ldkv, H * (dk + dv));
  B200_CHECK_ARG(aligned16(q) && aligned16(kv) && aligned16(out), "%s: pointers must be 16-byte aligned", what);
  B200_CHECK_ARG(H <= 65535 && B <= 65535, "%s: B=%d, H=%d exceed the grid", what, B, H);
  if (check_overlap) {
    const long long out_b = (long long)B * Nq * H * dv * 2, q_b = (((long long)B * Nq - 1) * ldq + (long long)H * dk) * 2,
                    kv_b = (((long long)B * Nk - 1) * ldkv + (long long)H * (dk + dv)) * 2;
    B200_CHECK_ARG(!overlap(out, out_b, q, q_b) && !overlap(out, out_b, kv, kv_b), "%s: out overlaps q or kv", what);
  }
  KvParams p{};
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.B = B;
  p.Nq = Nq;
  p.Nk = Nk;
  p.Ik = H * dk;
  p.Iv = H * dv;
  p.scale_log2e = scale * 1.4426950408889634f;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dk * 1000 + dv) {
    case 32032: return launch_kv_t<32, 32>(q, ldq, kv, ldkv, p, H, st);
    case 64064: return launch_kv_t<64, 64>(q, ldq, kv, ldkv, p, H, st);
    case 80080: return launch_kv_t<80, 80>(q, ldq, kv, ldkv, p, H, st);
    case 128128: return launch_kv_t<128, 128>(q, ldq, kv, ldkv, p, H, st);
    case 16032: return launch_kv_t<16, 32>(q, ldq, kv, ldkv, p, H, st);
    case 16064: return launch_kv_t<16, 64>(q, ldq, kv, ldkv, p, H, st);
    case 32064: return launch_kv_t<32, 64>(q, ldq, kv, ldkv, p, H, st);
    case 48032: return launch_kv_t<48, 32>(q, ldq, kv, ldkv, p, H, st);
    case 48064: return launch_kv_t<48, 64>(q, ldq, kv, ldkv, p, H, st);
    case 64032: return launch_kv_t<64, 32>(q, ldq, kv, ldkv, p, H, st);
    default: B200_CHECK_ARG(false, "%s: dk=%d, dv=%d not built", what, dk, dv);
  }
}

extern "C" int b200vit_attention_kv(const void* q, int64_t ldq, const void* kv, int64_t ldkv, void* out, int B, int Nq,
                                    int Nk, int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(head_width_ok(dh), "attention_kv: dim_head=%d not supported by this build (32, 64, 80 or 128)", dh);
  return attention_kv_impl("attention_kv", q, ldq, kv, ldkv, out, B, Nq, Nk, H, dh, dh, scale, stream);
}

extern "C" int b200vit_attention_kv_lens(const void* q, int64_t ldq, const void* kv, int64_t ldkv, void* out, int B,
                                         int Nq, int Nk, const int32_t* nk_dev, int H, int dh, float scale,
                                         void* stream) {
  B200_CHECK_ARG(nk_dev, "attention_kv_lens: null key counts");
  B200_CHECK_ARG(head_width_ok(dh), "attention_kv_lens: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(q && kv && out, "attention_kv_lens: null pointer");
  B200_CHECK_ARG(B > 0 && Nq > 0 && Nk > 0 && H > 0, "attention_kv_lens: bad shape B=%d Nq=%d Nk=%d H=%d", B, Nq, Nk,
                 H);
  B200_CHECK_ARG(Nk <= B200VIT_ATTN_KV_MAX_KEYS, "attention_kv_lens: Nk=%d > %d", Nk, B200VIT_ATTN_KV_MAX_KEYS);
  B200_CHECK_ARG(ldq >= (int64_t)H * dh && ldq % 8 == 0, "attention_kv_lens: ldq=%lld must be a multiple of 8 and >= %d",
                 (long long)ldq, H * dh);
  B200_CHECK_ARG(ldkv >= (int64_t)H * 2 * dh && ldkv % 8 == 0,
                 "attention_kv_lens: ldkv=%lld must be a multiple of 8 and >= %d", (long long)ldkv, 2 * H * dh);
  B200_CHECK_ARG(aligned16(q) && aligned16(kv) && aligned16(out), "attention_kv_lens: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535 && B <= 65535, "attention_kv_lens: B=%d, H=%d exceed the grid", B, H);
  const long long out_b = (long long)B * Nq * H * dh * 2, q_b = (((long long)B * Nq - 1) * ldq + (long long)H * dh) * 2,
                  kv_b = (((long long)B * Nk - 1) * ldkv + 2LL * H * dh) * 2;
  B200_CHECK_ARG(!overlap(out, out_b, q, q_b) && !overlap(out, out_b, kv, kv_b), "attention_kv_lens: out overlaps q or kv");
  KvParams p{};
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.B = B;
  p.Nq = Nq;
  p.Nk = Nk;
  p.Ik = H * dh;
  p.Iv = H * dh;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.nk = nk_dev;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: return launch_kv_t<32, 32, true>(q, ldq, kv, ldkv, p, H, st);
    case 80: return launch_kv_t<80, 80, true>(q, ldq, kv, ldkv, p, H, st);
    case 128: return launch_kv_t<128, 128, true>(q, ldq, kv, ldkv, p, H, st);
    default: return launch_kv_t<64, 64, true>(q, ldq, kv, ldkv, p, H, st);
  }
}

extern "C" int b200vit_attention_kv_ex(const void* q, int64_t ldq, const void* kv, int64_t ldkv, void* out, int B,
                                       int Nq, int Nk, int H, int dk, int dv, float scale, void* stream) {
  B200_CHECK_ARG(dk == 16 || dk == 32 || dk == 48 || dk == 64,
                 "attention_kv_ex: dk=%d not supported by this build (16, 32, 48 or 64)", dk);
  B200_CHECK_ARG(dv == 32 || dv == 64, "attention_kv_ex: dv=%d not supported by this build (32 or 64)", dv);
  return attention_kv_impl("attention_kv_ex", q, ldq, kv, ldkv, out, B, Nq, Nk, H, dk, dv, scale, stream, true);
}

extern "C" int b200vit_merge_patches_ln(const float* x, int64_t M, const float* gamma, const float* beta,
                                        void* out_bf16, int64_t ldo, int B, int gh, int gw, int C, int p, float eps,
                                        void* stream) {
  B200_CHECK_ARG(x && gamma && beta && out_bf16, "merge_patches_ln: null pointer");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && C > 0 && p > 0, "merge_patches_ln: bad shape B=%d h=%d w=%d C=%d p=%d",
                 B, gh, gw, C, p);
  B200_CHECK_ARG(gh % p == 0 && gw % p == 0, "merge_patches_ln: the %d x %d grid is not divisible by p=%d", gh, gw, p);
  B200_CHECK_ARG(M == (int64_t)B * gh * gw, "merge_patches_ln: x has %lld rows, %lld expected", (long long)M,
                 (long long)B * gh * gw);
  B200_CHECK_ARG(C % 4 == 0, "merge_patches_ln: C=%d must be a multiple of 4", C);
  B200_CHECK_ARG(ldo >= (int64_t)p * p * C && ldo % 8 == 0,
                 "merge_patches_ln: ldo=%lld must be a multiple of 8 and >= %lld", (long long)ldo,
                 (long long)p * p * C);
  B200_CHECK_ARG(aligned16(x) && aligned16(gamma) && aligned16(beta) && aligned16(out_bf16),
                 "merge_patches_ln: pointers must be 16-byte aligned");
  const long long rows = (long long)B * (gh / p) * (gw / p);
  B200_CHECK_ARG((rows + 7) / 8 <= 0x7fffffffLL, "merge_patches_ln: %lld rows exceed the grid", rows);
  merge_patches_ln_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, gamma, beta, reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, (int)rows, gh, gw, C, p, eps);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_peg(const float* x, int64_t M, const float* w, const float* bias, float* y, int B, int gh,
                           int gw, int C, int k, void* stream) {
  B200_CHECK_ARG(x && w && bias && y, "peg: null pointer");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && C > 0, "peg: bad shape B=%d h=%d w=%d C=%d", B, gh, gw, C);
  B200_CHECK_ARG(k == 1 || k == 3 || k == 5 || k == 7, "peg: kernel size %d not built (1, 3, 5 or 7)", k);
  B200_CHECK_ARG(M == (int64_t)B * gh * gw, "peg: x has %lld rows, %lld expected", (long long)M,
                 (long long)B * gh * gw);
  B200_CHECK_ARG(C % 4 == 0, "peg: C=%d must be a multiple of 4", C);
  B200_CHECK_ARG(x != y, "peg: y must not be x (every token reads its neighbours)");
  B200_CHECK_ARG(aligned16(x) && aligned16(w) && aligned16(bias) && aligned16(y),
                 "peg: pointers must be 16-byte aligned");
  const long long total4 = M * (C / 4);
  B200_CHECK_ARG((total4 + 255) / 256 <= 0x7fffffffLL, "peg: %lld elements exceed the grid", total4 * 4);
  peg_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, w, bias, y,
                                                                                                   total4, gh, gw, C, k);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
