// Kernels of ScalableViT (reference scalable_vit.py), for sm_90a.  The token map of a stage is kept channels-last,
// token (b, y, x) at row (b*gh + y)*gw + x.  The sub-sampled-key attention of the SSA is b200vit_attention_kv_ex in
// twins.cu.
//   b200vit_attention_iwsa   attention inside wh x ww windows of the map, plus the local interactive module's output
//                            (InteractiveWindowedSelfAttention, scalable_vit.py:155-194)
//
// attention_iwsa: one CTA = two warpgroups = 128 query rows of one (window, head), 64 rows per warpgroup.  The window's
// keys and values stream through a ring of IW_RING block slots of 64 keys, loaded IW_RING - 1 blocks ahead by
// cp.async.  Every row is gathered from its map-order address (no rearranged copy of the windows exists), rows past
// the window are zero-filled without a read.  The shape the tiling is for: whole-map windows of 4096 tokens at
// dk = dv = 32 and 2 heads (the README ScalableViT-S, stage 1), 32 query tiles per (image, head), so each key block
// is read from L2 by 32 CTAs.  Per block: S = Q K^T with wgmma, keys past the window masked to -inf, the online
// softmax of attention.cu in fp32, O += P V with wgmma.  The output is fma(O, 1 / l, lim) in fp32, rounded to bf16 once.
#include "tile64.cuh"
#include "host_util.h"

namespace b200 {

using namespace tile64;

constexpr int IW_THREADS = 256;
constexpr int IW_RING = 4;

struct IwsaParams {
  const __nv_bfloat16* qkv;
  const __nv_bfloat16* lim;
  __nv_bfloat16* out;
  long long ld;            // row stride of qkv
  int gh, gw, wh, ww;
  int X, Y;                // windows along y and x
  int n, nqt;              // tokens of a window, 128-row query tiles of a window
  int Ik, Iv;              // H * dk, H * dv
  float scale_log2e;
};

// rows [r0, r0 + 64) of the window (map rows from row_of, negative: zero-filled) into the operand block at `base`,
// D columns from `col`; all IW_THREADS threads issue their share of the 16-byte pieces
template <int D, typename RowFn>
__device__ __forceinline__ void iw_load(uint32_t base, const __nv_bfloat16* qkv, long long ld, int col, int r0,
                                        RowFn row_of, int tid) {
  constexpr int P = D / 8;
  for (int i = tid; i < ROWS * P; i += IW_THREADS) {
    const int r = i / P, c = i - r * P;
    const long long row = row_of(r0 + r);
    const bool ok = row >= 0;
    cp_async16(piece_addr<D>(base, r, c), ok ? qkv + row * ld + col + 8 * c : qkv, ok);
  }
}

// this thread's output row half rh: fma(O, inv, lim) in fp32, one rounding to bf16; op / lp: the row's first column
template <int DV>
__device__ __forceinline__ void store_rows_lim(const float (&o)[Slabs<DV>::N64 > 0 ? Slabs<DV>::N64 : 1][32],
                                               const float (&o16)[Slabs<DV>::N16 > 0 ? Slabs<DV>::N16 : 1][8],
                                               __nv_bfloat16* op, const __nv_bfloat16* lp, int rh, float inv) {
  using S = Slabs<DV>;
  auto put = [&](int col, float a, float b) {
    const float2 l = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(lp + col));
    *reinterpret_cast<uint32_t*>(op + col) = pack_bf16x2(fmaf(a, inv, l.x), fmaf(b, inv, l.y));
  };
#pragma unroll
  for (int c = 0; c < S::N64; ++c)
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) put(64 * c + jj * 8, o[c][4 * jj + 2 * rh], o[c][4 * jj + 2 * rh + 1]);
#pragma unroll
  for (int c = 0; c < S::N16; ++c)
#pragma unroll
    for (int jj = 0; jj < 2; ++jj)
      put(64 * S::N64 + 16 * c + jj * 8, o16[c][4 * jj + 2 * rh], o16[c][4 * jj + 2 * rh + 1]);
}

// CTAs per SM the registers are bounded for.  Both products are waited on inside each key block, so co-resident CTAs
// are what hides a block's latency: 3 (at most 80 registers) where that costs no spill, dk = 32 or 64 with dv = 32
// (the README shapes; 90 registers unbounded, i.e. 2 CTAs), else 2
template <int DK, int DV>
constexpr int iw_min_ctas() { return DV == 32 && DK % 32 == 0 ? 3 : 2; }

template <int DK, int DV>
__global__ void __launch_bounds__(IW_THREADS, iw_min_ctas<DK, DV>())
attention_iwsa_kernel(const IwsaParams p) {
  using SK = Slabs<DK>;
  using SV = Slabs<DV>;
  constexpr int N64 = SV::N64, N16 = SV::N16;
  constexpr int SLOT = SK::OP + SV::OP;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // Q: two operand blocks (one per warpgroup); then IW_RING slots of K | V
  const uint32_t sq0 = smem_u32(smem), slot0 = sq0 + 2 * SK::OP;

  const int h = blockIdx.y;
  const int win = blockIdx.x / p.nqt, qt = blockIdx.x - win * p.nqt;
  const int b = win / (p.X * p.Y), wi = (win / p.Y) % p.X, wj = win % p.Y;
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  const int n = p.n, nkb = (n + 63) / 64, q0 = qt * 128;

  // token t of the window -> its row of the map, -1 past the window
  const long long row0 = ((long long)b * p.gh + wi * p.wh) * p.gw + wj * p.ww;
  auto row_of = [&](int t) -> long long {
    if (t >= n) return -1;
    const int u = t / p.ww;
    return row0 + u * p.gw + (t - u * p.ww);
  };
  auto load_kv = [&](int j) {
    const uint32_t dst = slot0 + (j % IW_RING) * SLOT;
    iw_load<DK>(dst, p.qkv, p.ld, p.Ik + h * DK, 64 * j, row_of, tid);
    iw_load<DV>(dst + SK::OP, p.qkv, p.ld, 2 * p.Ik + h * DV, 64 * j, row_of, tid);
  };

  // groups: Q with block 0, then one per block; a group is committed for every block index, loaded or not, so that
  // wait_group<IW_RING - 2> at block kb always means "block kb has landed"
  iw_load<DK>(sq0, p.qkv, p.ld, h * DK, q0, row_of, tid);
  iw_load<DK>(sq0 + SK::OP, p.qkv, p.ld, h * DK, q0 + 64, row_of, tid);
#pragma unroll
  for (int j = 0; j < IW_RING - 1; ++j) {
    if (j < nkb) load_kv(j);
    cp_async_commit();
  }

  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[N64 > 0 ? N64 : 1][32], o16[N16 > 0 ? N16 : 1][8];
  zero_acc<DV>(o, o16);
  const uint32_t sq = sq0 + wg * SK::OP;

  for (int kb = 0; kb < nkb; ++kb) {
    cp_async_wait<IW_RING - 2>();  // this thread's pieces of block kb (and of Q) have landed
    fence_proxy_async_smem();      // ... and are visible to wgmma
    __syncthreads();               // ... as are every other thread's; every thread is done with block kb - 1
    if (kb + IW_RING - 1 < nkb) load_kv(kb + IW_RING - 1);   // into the slot of block kb - 1
    cp_async_commit();
    const uint32_t sk = slot0 + (kb % IW_RING) * SLOT, sv = sk + SK::OP;

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
        s[4 * jj + e] = key0 + 8 * jj + (e & 1) < n ? s[4 * jj + e] * p.scale_log2e : -INFINITY;
        mn[rh] = fmaxf(mn[rh], s[4 * jj + e]);
      }
    quad_max(mn);
    float alpha[2];
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      // every block holds at least one key of the window, so mn is finite unless the scores are not
      alpha[rh] = fast_ex2(m[rh] - mn[rh]);
      m[rh] = mn[rh];
      l[rh] *= alpha[rh];
    }
    tile_exp2(s, m, l);  // this thread's keys only: l is summed over the four lanes of the row after the last block
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
  cp_async_wait<0>();  // no copy is left in flight when the CTA exits (the trailing groups are empty)

  quad_sum(l);
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int t = q0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * rh;
    if (t >= n) continue;
    const long long off = row_of(t) * p.Iv + h * DV + 2 * (lane & 3);
    store_rows_lim<DV>(o, o16, p.out + off, p.lim + off, rh, 1.0f / l[rh]);
  }
}

template <int DK, int DV>
static int launch_iwsa_t(const IwsaParams& p, int H, long long ctas, cudaStream_t stream) {
  using SK = Slabs<DK>;
  using SV = Slabs<DV>;
  const int bytes = 2 * SK::OP + IW_RING * (SK::OP + SV::OP) + 1024;
  auto kern = attention_iwsa_kernel<DK, DV>;
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3((unsigned)ctas, H), IW_THREADS, bytes, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace b200

using namespace b200;

static bool al16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

static bool overlap(const void* a, long long a_bytes, const void* b, long long b_bytes) {
  const uintptr_t p = reinterpret_cast<uintptr_t>(a), q = reinterpret_cast<uintptr_t>(b);
  return p < q + (uintptr_t)b_bytes && q < p + (uintptr_t)a_bytes;
}

extern "C" int b200vit_attention_iwsa(const void* qkv, int64_t ld, const void* lim, void* out, int B, int gh, int gw,
                                      int wh, int ww, int H, int dk, int dv, float scale, void* stream) {
  B200_CHECK_ARG(qkv && lim && out, "attention_iwsa: null pointer");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && wh > 0 && ww > 0 && H > 0,
                 "attention_iwsa: bad shape B=%d h=%d w=%d window %d x %d H=%d", B, gh, gw, wh, ww, H);
  B200_CHECK_ARG(dk == 16 || dk == 32 || dk == 48 || dk == 64,
                 "attention_iwsa: dk=%d not supported by this build (16, 32, 48 or 64)", dk);
  B200_CHECK_ARG(dv == 32 || dv == 64, "attention_iwsa: dv=%d not supported by this build (32 or 64)", dv);
  B200_CHECK_ARG(gh % wh == 0 && gw % ww == 0, "attention_iwsa: the %d x %d map is not divisible by the %d x %d window",
                 gh, gw, wh, ww);
  B200_CHECK_ARG((long long)wh * ww <= B200VIT_ATTN_KV_MAX_KEYS, "attention_iwsa: a %d x %d window has more than %d tokens",
                 wh, ww, B200VIT_ATTN_KV_MAX_KEYS);
  const long long I = (long long)H * (2 * dk + dv), Iv = (long long)H * dv;
  B200_CHECK_ARG(ld >= I && ld % 8 == 0, "attention_iwsa: ld=%lld must be a multiple of 8 and >= %lld", (long long)ld,
                 I);
  const long long rows = (long long)B * gh * gw;
  const long long nwin = (long long)B * (gh / wh) * (gw / ww), nqt = ((long long)wh * ww + 127) / 128;
  B200_CHECK_ARG(H <= 65535 && nwin * nqt <= 0x7fffffffLL, "attention_iwsa: %lld windows x %d heads exceed the grid",
                 nwin, H);
  B200_CHECK_ARG(al16(qkv) && al16(lim) && al16(out), "attention_iwsa: pointers must be 16-byte aligned");
  B200_CHECK_ARG(!overlap(out, rows * Iv * 2, qkv, ((rows - 1) * ld + I) * 2) && !overlap(out, rows * Iv * 2, lim, rows * Iv * 2),
                 "attention_iwsa: out overlaps qkv or lim");
  IwsaParams p{};
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv);
  p.lim = reinterpret_cast<const __nv_bfloat16*>(lim);
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ld = ld;
  p.gh = gh;
  p.gw = gw;
  p.wh = wh;
  p.ww = ww;
  p.X = gh / wh;
  p.Y = gw / ww;
  p.n = wh * ww;
  p.nqt = (int)nqt;
  p.Ik = H * dk;
  p.Iv = H * dv;
  p.scale_log2e = scale * 1.4426950408889634f;
  const long long ctas = nwin * nqt;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dk * 1000 + dv) {
    case 16032: return launch_iwsa_t<16, 32>(p, H, ctas, st);
    case 16064: return launch_iwsa_t<16, 64>(p, H, ctas, st);
    case 32032: return launch_iwsa_t<32, 32>(p, H, ctas, st);
    case 32064: return launch_iwsa_t<32, 64>(p, H, ctas, st);
    case 48032: return launch_iwsa_t<48, 32>(p, H, ctas, st);
    case 48064: return launch_iwsa_t<48, 64>(p, H, ctas, st);
    case 64032: return launch_iwsa_t<64, 32>(p, H, ctas, st);
    default: return launch_iwsa_t<64, 64>(p, H, ctas, st);
  }
}
