// Kernels of the hierarchical, window-attention models (Twins-SVT, reference twins_svt.py), for sm_90a.  The token map
// of a stage is kept token-major: x[B*gh*gw, C], token (b, y, x) at row (b*gh + y)*gw + x.
//   b200vit_attention_window   softmax attention inside non-overlapping p x p windows of the map (twins_svt.py:85-120)
//   b200vit_attention_kv       every query of an image against that image's keys / values, which come from another
//                              buffer and have another length (twins_svt.py:122-157: the sub-sampled keys)
//   b200vit_merge_patches_ln   p x p patch merging + LayerNorm over the merged features (twins_svt.py:59-75)
//   b200vit_peg                depthwise k x k convolution plus identity (twins_svt.py:77-83)
//
// attention_window is the tile scheme of axial.cu with a 2-D gather: one CTA = one warpgroup = one 64-row tile of one
// head that holds spy x spx whole windows of one image.  Thread 0 loads Q, K and V with one TMA box per slab over the
// 4-D view (column, x, y, b) of qkv: the box is (p spx) tokens wide and (p spy) tall, box row r = iy * (p spx) + ix;
// tokens outside the map are zero-filled.  S = Q K^T (64 x 64) with wgmma, a block-diagonal mask (same window) in
// registers, a plain fp32 softmax (every key of a row is in the tile) and O = P V with wgmma.  A tile never holds two
// images.  Windows that share a tile (p*p <= 32) meet each other's V rows in O = P V with probability exactly 0, so a
// finite change in one window leaves the others bit-identical; a NaN or Inf stays within its image, and within its
// window when p*p > 32 (one window per tile).
//
// attention_kv: one CTA = two warpgroups = one (image, head) and a strided share of its 128-row query tiles, 64 rows
// per warpgroup.  Keys and values are cut in blocks of 64 that thread 0 loads with TMA over the 3-D view (column, key,
// image) of kv, keys past Nk zero-filled.  Most of the work of a CTA is on the query side (Nq >> Nk in Twins-SVT: 3136
// queries against 64 keys), so when all key blocks of the (image, head) fit the CTA's shared memory they are loaded
// once and every query tile of the CTA loops over them; otherwise they stream through a ring of 4 block slots, loaded
// 3 blocks ahead, once per query tile.  Per block: S = Q K^T with wgmma, keys past Nk masked to -inf, the online
// softmax of attention.cu in fp32, O += P V with wgmma (P from registers, V as the transposed B operand).  The
// resident / streaming choice and the CTA count are untuned: no measurement preceded them.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int TW_ROWS = 64;
constexpr int TW_THREADS = 128;

// One operand block of 64 rows: N64 slabs 64 columns wide (128B swizzle), then N16 slabs 16 columns wide (32B swizzle).
template <int DH>
struct Slabs {
  static constexpr int N64 = DH / 64;
  static constexpr int N16 = (DH % 64) / 16;
  static_assert(N64 * 64 + N16 * 16 == DH, "dim_head must be a multiple of 16");
  static constexpr int S64 = TW_ROWS * 128;
  static constexpr int S16 = TW_ROWS * 32;
  static constexpr int OP = N64 * S64 + N16 * S16;
};

// S[64 x 64] = Q K^T over the slabs of one operand block each
template <int DH>
__device__ __forceinline__ void qk_mma(float (&s)[32], uint32_t sq, uint32_t sk) {
  using S = Slabs<DH>;
#pragma unroll
  for (int c = 0; c < S::N64; ++c)
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_m64n64k16(s, make_wgmma_desc(sq + c * S::S64, 1024, WGMMA_SW128) + 2 * k,
                      make_wgmma_desc(sk + c * S::S64, 1024, WGMMA_SW128) + 2 * k, c != 0 || k != 0);
#pragma unroll
  for (int c = 0; c < S::N16; ++c)
    wgmma_m64n64k16(s, make_wgmma_desc(sq + S::N64 * S::S64 + c * S::S16, 256, WGMMA_SW32),
                    make_wgmma_desc(sk + S::N64 * S::S64 + c * S::S16, 256, WGMMA_SW32), S::N64 != 0 || c != 0);
}

// O[64 x DH] += P V, P the 64 x 64 probabilities in this thread's S registers, V one operand block
template <int DH>
__device__ __forceinline__ void pv_mma(float (&o)[Slabs<DH>::N64 > 0 ? Slabs<DH>::N64 : 1][32],
                                       float (&o16)[Slabs<DH>::N16 > 0 ? Slabs<DH>::N16 : 1][8], const float (&s)[32],
                                       uint32_t sv) {
  using S = Slabs<DH>;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                           pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
#pragma unroll
    for (int c = 0; c < S::N64; ++c)
      wgmma_m64n64k16_rs_tb(o[c], a, make_wgmma_desc_lbo(sv + c * S::S64 + kk * 2048, 1024, 1024, WGMMA_SW128));
#pragma unroll
    for (int c = 0; c < S::N16; ++c)
      wgmma_m64n16k16_rs_tb(o16[c], a,
                            make_wgmma_desc_lbo(sv + S::N64 * S::S64 + c * S::S16 + kk * 512, 256, 256, WGMMA_SW32));
  }
}

// this thread's two output rows (rh) of O, scaled by inv[rh], to op[rh] (the row's first column of this head)
template <int DH>
__device__ __forceinline__ void store_rows(const float (&o)[Slabs<DH>::N64 > 0 ? Slabs<DH>::N64 : 1][32],
                                           const float (&o16)[Slabs<DH>::N16 > 0 ? Slabs<DH>::N16 : 1][8],
                                           __nv_bfloat16* op, int rh, float inv) {
  using S = Slabs<DH>;
#pragma unroll
  for (int c = 0; c < S::N64; ++c)
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
      *reinterpret_cast<uint32_t*>(op + 64 * c + jj * 8) =
          pack_bf16x2(o[c][4 * jj + 2 * rh] * inv, o[c][4 * jj + 2 * rh + 1] * inv);
#pragma unroll
  for (int c = 0; c < S::N16; ++c)
#pragma unroll
    for (int jj = 0; jj < 2; ++jj)
      *reinterpret_cast<uint32_t*>(op + 64 * S::N64 + 16 * c + jj * 8) =
          pack_bf16x2(o16[c][4 * jj + 2 * rh] * inv, o16[c][4 * jj + 2 * rh + 1] * inv);
}

// ------------------------------------------------------------------------------------------------ attention_window
struct WindowParams {
  __nv_bfloat16* out;
  int B, gh, gw, p, I;     // I = H * dh
  int spx, spy;            // windows per tile along x and y
  int tiles_x, tiles_y;
  float scale_log2e;
};

template <int DH>
__global__ void __launch_bounds__(TW_THREADS)
attention_window_kernel(const __grid_constant__ CUtensorMap tm64, const __grid_constant__ CUtensorMap tm16,
                        const WindowParams p) {
  using S = Slabs<DH>;
  constexpr int N64 = S::N64, N16 = S::N16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 3 * S::OP);

  const int h = blockIdx.y;
  const int tx = blockIdx.x % p.tiles_x, ty = (blockIdx.x / p.tiles_x) % p.tiles_y;
  const int b0 = blockIdx.x / (p.tiles_x * p.tiles_y);
  const int bw = p.p * p.spx, bh = p.p * p.spy;  // the box, in tokens
  const int x0 = tx * bw, y0 = ty * bh;
  const int rows = bw * bh;                       // <= 64
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // rows beyond the box: their keys are masked, but V meets a zero probability in O = P V and must be finite
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int o = 0; o < 3; ++o) {
#pragma unroll
    for (int c = 0; c < N64; ++c) {
      uint4* sl = reinterpret_cast<uint4*>(smem + o * S::OP + c * S::S64);
      for (int i = rows * 8 + tid; i < TW_ROWS * 8; i += TW_THREADS) sl[i] = z;
    }
#pragma unroll
    for (int c = 0; c < N16; ++c) {
      uint4* sl = reinterpret_cast<uint4*>(smem + o * S::OP + N64 * S::S64 + c * S::S16);
      for (int i = rows * 2 + tid; i < TW_ROWS * 2; i += TW_THREADS) sl[i] = z;
    }
  }
  fence_proxy_async_smem();
  if (tid == 0) {
    tma_prefetch_desc(N64 ? &tm64 : &tm16);
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 3 * rows * DH * 2);  // zero-filled elements count too
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      const int col = o * p.I + h * DH;
#pragma unroll
      for (int c = 0; c < N64; ++c) tma_load_4d(smem + o * S::OP + c * S::S64, &tm64, bar, col + 64 * c, x0, y0, b0);
#pragma unroll
      for (int c = 0; c < N16; ++c)
        tma_load_4d(smem + o * S::OP + N64 * S::S64 + c * S::S16, &tm16, bar, col + 64 * N64 + 16 * c, x0, y0, b0);
    }
  }

  // this thread's rows r = 16 warp + lane/4 + 8 rh and key columns c = 8 jj + 2 (lane % 4) + e1 (wgmma m64 layout):
  // the window of each within the tile, -1 for a key outside the box or the map
  int rwin[2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int r = warp * 16 + (lane >> 2) + 8 * rh;
    rwin[rh] = ((r / bw) / p.p) * p.spx + (r % bw) / p.p;
  }
  int cwin[16];
#pragma unroll
  for (int ci = 0; ci < 16; ++ci) {
    const int c = 8 * (ci >> 1) + 2 * (lane & 3) + (ci & 1);
    const int iy = c / bw, ix = c % bw;
    cwin[ci] = (c < rows && x0 + ix < p.gw && y0 + iy < p.gh) ? (iy / p.p) * p.spx + ix / p.p : -1;
  }

  mbar_wait(bar, 0);

  float s[32];
  const uint32_t sq = smem_u32(smem), sk = sq + S::OP, sv = sq + 2 * S::OP;
  wgmma_fence();
  qk_mma<DH>(s, sq, sk);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);

  // plain softmax in log2 units; s[4 jj + e]: row half e >> 1, key column index ci = 2 jj + (e & 1)
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int ci = 2 * jj + (e & 1), rh = e >> 1;
      s[4 * jj + e] = cwin[ci] == rwin[rh] ? s[4 * jj + e] * p.scale_log2e : -INFINITY;
      mx[rh] = fmaxf(mx[rh], s[4 * jj + e]);
    }
  float l[2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 1));
    mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 2));
    l[rh] = 0.f;
  }
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int rh = e >> 1;
      // a row outside the map has no key (mx = -inf): probability 0 everywhere, never stored
      const float v = mx[rh] != -INFINITY ? fast_ex2(s[4 * jj + e] - mx[rh]) : 0.f;
      s[4 * jj + e] = v;
      l[rh] += v;
    }
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 1);
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 2);
    l[rh] = l[rh] > 0.f ? 1.0f / l[rh] : 0.f;
  }

  float o[N64 > 0 ? N64 : 1][32], o16[N16 > 0 ? N16 : 1][8];
#pragma unroll
  for (int c = 0; c < N64; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
#pragma unroll
  for (int c = 0; c < N16; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) o16[c][i] = 0.f;
  wgmma_fence();
  pv_mma<DH>(o, o16, s, sv);
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < N64; ++c) fence_regs(o[c]);
#pragma unroll
  for (int c = 0; c < N16; ++c) fence_regs(o16[c]);

#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int r = warp * 16 + (lane >> 2) + 8 * rh;
    const int y = y0 + r / bw, x = x0 + r % bw;
    if (r >= rows || x >= p.gw || y >= p.gh) continue;
    store_rows<DH>(o, o16, p.out + (((long long)b0 * p.gh + y) * p.gw + x) * p.I + h * DH + 2 * (lane & 3), rh, l[rh]);
  }
}

// Tensor maps over the 4-D view (column, x, y, b) of qkv: boxes of 64 columns (128B swizzle) and 16 columns (32B
// swizzle) by (p spx) x (p spy) x 1 tokens.  A kind the head does not use gets a copy of the other (never read).
template <int DH>
static int launch_window_t(const void* qkv, const WindowParams& p, int H, int tiles, cudaStream_t stream) {
  using S = Slabs<DH>;
  CUtensorMap tm[2];
  const uint64_t ld = (uint64_t)3 * p.I;
  const uint64_t dims[4] = {ld, (uint64_t)p.gw, (uint64_t)p.gh, (uint64_t)p.B};
  const uint64_t strides[3] = {ld * 2, ld * 2 * p.gw, ld * 2 * p.gw * p.gh};
  const uint32_t bw = (uint32_t)(p.p * p.spx), bh = (uint32_t)(p.p * p.spy);
  const uint32_t box64[4] = {64, bw, bh, 1};
  const uint32_t box16[4] = {16, bw, bh, 1};
  int rc = 0;
  if (S::N64) rc = encode_tmap_bf16(&tm[0], qkv, 4, dims, strides, box64);
  if (!rc && S::N16) rc = encode_tmap_bf16_sw(&tm[1], qkv, 4, dims, strides, box16, 32);
  if (rc) return rc;
  if (!S::N16) tm[1] = tm[0];
  if (!S::N64) tm[0] = tm[1];
  auto kern = attention_window_kernel<DH>;
  const int bytes = 3 * S::OP + 8 + 1024;  // barrier; slack for 1024B alignment
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3(tiles, H), TW_THREADS, bytes, stream>>>(tm[0], tm[1], p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------ attention_kv
constexpr int KV_THREADS = 256;
constexpr int KV_RING = 4;             // block slots of the streaming mode
constexpr int KV_SMEM = 200 * 1024;    // what a CTA may hold: the query tile and the resident key / value blocks
constexpr int KV_MAX_SLOTS = 16;

template <int DH>
constexpr int kv_resident_slots() {
  const int n = (KV_SMEM - 2 * Slabs<DH>::OP) / (2 * Slabs<DH>::OP);
  return n < KV_MAX_SLOTS ? n : KV_MAX_SLOTS;
}

struct KvParams {
  __nv_bfloat16* out;
  int B, Nq, Nk, I;
  int slots;               // block slots in shared memory; all blocks resident iff ceil(Nk / 64) <= slots
  float scale_log2e;
};

template <int DH>
__global__ void __launch_bounds__(KV_THREADS)
attention_kv_kernel(const __grid_constant__ CUtensorMap q64, const __grid_constant__ CUtensorMap q16,
                    const __grid_constant__ CUtensorMap kv64, const __grid_constant__ CUtensorMap kv16,
                    const KvParams p) {
  using S = Slabs<DH>;
  constexpr int N64 = S::N64, N16 = S::N16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // Q: two operand blocks (one per warpgroup); then per slot K | V; then the barriers: Q, one per slot
  uint8_t* slot0 = smem + 2 * S::OP;
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(slot0 + (size_t)p.slots * 2 * S::OP);
  uint64_t* bar_kv = bar_q + 1;

  const int h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  const int nqt = (p.Nq + 127) / 128, nkb = (p.Nk + 63) / 64;
  const bool resident = nkb <= p.slots;

  if (tid == 0) {
    tma_prefetch_desc(N64 ? &q64 : &q16);
    tma_prefetch_desc(N64 ? &kv64 : &kv16);
    mbar_init(bar_q, 1);
    for (int i = 0; i < p.slots; ++i) mbar_init(bar_kv + i, 1);
    fence_mbar_init();
  }

  auto load_block = [&](int j) {  // thread 0: keys [64 j, 64 j + 64) of image b into slot j % slots
    const int sl = j % p.slots;
    uint8_t* dst = slot0 + (size_t)sl * 2 * S::OP;
    mbar_arrive_expect_tx(bar_kv + sl, 2 * TW_ROWS * DH * 2);
#pragma unroll
    for (int o = 0; o < 2; ++o) {
      const int col = o * p.I + h * DH;
#pragma unroll
      for (int c = 0; c < N64; ++c) tma_load_3d(dst + o * S::OP + c * S::S64, &kv64, bar_kv + sl, col + 64 * c, 64 * j, b);
#pragma unroll
      for (int c = 0; c < N16; ++c)
        tma_load_3d(dst + o * S::OP + N64 * S::S64 + c * S::S16, &kv16, bar_kv + sl, col + 64 * N64 + 16 * c, 64 * j, b);
    }
  };

  uint32_t q_phase = 0, kv_phase = 0;  // kv_phase: one bit per slot
  bool first = true;
  for (int qt = blockIdx.x; qt < nqt; qt += gridDim.x, first = false) {
    const int q0 = qt * 128;
    __syncthreads();  // the barriers are initialised; every thread is done with the previous tile's Q (and slots)
    if (tid == 0) {
      mbar_arrive_expect_tx(bar_q, 2 * TW_ROWS * DH * 2);
#pragma unroll
      for (int w = 0; w < 2; ++w) {
#pragma unroll
        for (int c = 0; c < N64; ++c) tma_load_3d(smem + w * S::OP + c * S::S64, &q64, bar_q, h * DH + 64 * c, q0 + 64 * w, b);
#pragma unroll
        for (int c = 0; c < N16; ++c)
          tma_load_3d(smem + w * S::OP + N64 * S::S64 + c * S::S16, &q16, bar_q, h * DH + 64 * N64 + 16 * c,
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
      const uint32_t sk = smem_u32(slot0) + sl * 2 * S::OP, sv = sk + S::OP;

      float s[32];
      wgmma_fence();
      qk_mma<DH>(s, sq, sk);
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
          s[4 * jj + e] = key0 + 8 * jj + (e & 1) < p.Nk ? s[4 * jj + e] * p.scale_log2e : -INFINITY;
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
      pv_mma<DH>(o, o16, s, sv);
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
      store_rows<DH>(o, o16, p.out + ((long long)b * p.Nq + q) * p.I + h * DH + 2 * (lane & 3), rh, 1.0f / l[rh]);
    }
  }
}

template <int DH>
static int launch_kv_t(const void* q, int64_t ldq, const void* kv, int64_t ldkv, KvParams p, int H,
                       cudaStream_t stream) {
  using S = Slabs<DH>;
  CUtensorMap tm[4];
  const uint64_t qdims[3] = {(uint64_t)p.I, (uint64_t)p.Nq, (uint64_t)p.B};
  const uint64_t qstr[2] = {(uint64_t)ldq * 2, (uint64_t)ldq * 2 * p.Nq};
  const uint64_t kdims[3] = {(uint64_t)2 * p.I, (uint64_t)p.Nk, (uint64_t)p.B};
  const uint64_t kstr[2] = {(uint64_t)ldkv * 2, (uint64_t)ldkv * 2 * p.Nk};
  const uint32_t box64[3] = {64, TW_ROWS, 1}, box16[3] = {16, TW_ROWS, 1};
  int rc = 0;
  if (S::N64) {
    rc = encode_tmap_bf16(&tm[0], q, 3, qdims, qstr, box64);
    if (!rc) rc = encode_tmap_bf16(&tm[2], kv, 3, kdims, kstr, box64);
  }
  if (!rc && S::N16) {
    rc = encode_tmap_bf16_sw(&tm[1], q, 3, qdims, qstr, box16, 32);
    if (!rc) rc = encode_tmap_bf16_sw(&tm[3], kv, 3, kdims, kstr, box16, 32);
  }
  if (rc) return rc;
  if (!S::N16) tm[1] = tm[0], tm[3] = tm[2];
  if (!S::N64) tm[0] = tm[1], tm[2] = tm[3];
  const int nkb = (p.Nk + 63) / 64, nqt = (p.Nq + 127) / 128;
  p.slots = nkb <= kv_resident_slots<DH>() ? nkb : KV_RING;
  const int bytes = (2 + 2 * p.slots) * S::OP + 8 * (1 + KV_MAX_SLOTS) + 1024;
  // enough CTAs to fill the device about twice; an (image, head) with resident keys is not split further than that
  const long long pairs = (long long)p.B * H;
  long long per = (2LL * num_sms() + pairs - 1) / pairs;
  if (per > nqt) per = nqt;
  if (per < 1) per = 1;
  auto kern = attention_kv_kernel<DH>;
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

extern "C" int b200vit_attention_window(const void* qkv, void* out, int B, int gh, int gw, int p, int H, int dh,
                                        float scale, void* stream) {
  B200_CHECK_ARG(qkv && out, "attention_window: null pointer");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && p > 0 && H > 0, "attention_window: bad shape B=%d h=%d w=%d p=%d H=%d", B,
                 gh, gw, p, H);
  B200_CHECK_ARG(head_width_ok(dh), "attention_window: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(p * p <= TW_ROWS, "attention_window: p=%d, a window of %d tokens must fit one %d-row tile", p, p * p,
                 TW_ROWS);
  B200_CHECK_ARG(gh % p == 0 && gw % p == 0, "attention_window: the %d x %d grid is not divisible into %d x %d windows",
                 gh, gw, p, p);
  B200_CHECK_ARG(aligned16(qkv) && aligned16(out), "attention_window: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535, "attention_window: H=%d exceeds the grid", H);
  WindowParams q{};
  q.out = reinterpret_cast<__nv_bfloat16*>(out);
  q.B = B;
  q.gh = gh;
  q.gw = gw;
  q.p = p;
  q.I = H * dh;
  const int fit = TW_ROWS / (p * p), wx = gw / p, wy = gh / p;
  q.spx = wx < fit ? wx : fit;
  q.spy = wy < fit / q.spx ? wy : fit / q.spx;
  q.tiles_x = (wx + q.spx - 1) / q.spx;
  q.tiles_y = (wy + q.spy - 1) / q.spy;
  const long long tiles = (long long)q.tiles_x * q.tiles_y * B;
  B200_CHECK_ARG(tiles <= 0x7fffffffLL, "attention_window: %lld tiles exceed the grid", tiles);
  q.scale_log2e = scale * 1.4426950408889634f;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: return launch_window_t<32>(qkv, q, H, (int)tiles, st);
    case 80: return launch_window_t<80>(qkv, q, H, (int)tiles, st);
    case 128: return launch_window_t<128>(qkv, q, H, (int)tiles, st);
    default: return launch_window_t<64>(qkv, q, H, (int)tiles, st);
  }
}

extern "C" int b200vit_attention_kv(const void* q, int64_t ldq, const void* kv, int64_t ldkv, void* out, int B, int Nq,
                                    int Nk, int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(q && kv && out, "attention_kv: null pointer");
  B200_CHECK_ARG(B > 0 && Nq > 0 && Nk > 0 && H > 0, "attention_kv: bad shape B=%d Nq=%d Nk=%d H=%d", B, Nq, Nk, H);
  B200_CHECK_ARG(head_width_ok(dh), "attention_kv: dim_head=%d not supported by this build (32, 64, 80 or 128)", dh);
  B200_CHECK_ARG(Nk <= B200VIT_ATTN_KV_MAX_KEYS, "attention_kv: Nk=%d > %d", Nk, B200VIT_ATTN_KV_MAX_KEYS);
  B200_CHECK_ARG(ldq >= (int64_t)H * dh && ldq % 8 == 0, "attention_kv: ldq=%lld must be a multiple of 8 and >= %d",
                 (long long)ldq, H * dh);
  B200_CHECK_ARG(ldkv >= (int64_t)2 * H * dh && ldkv % 8 == 0,
                 "attention_kv: ldkv=%lld must be a multiple of 8 and >= %d", (long long)ldkv, 2 * H * dh);
  B200_CHECK_ARG(aligned16(q) && aligned16(kv) && aligned16(out), "attention_kv: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535 && B <= 65535, "attention_kv: B=%d, H=%d exceed the grid", B, H);
  KvParams p{};
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.B = B;
  p.Nq = Nq;
  p.Nk = Nk;
  p.I = H * dh;
  p.scale_log2e = scale * 1.4426950408889634f;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: return launch_kv_t<32>(q, ldq, kv, ldkv, p, H, st);
    case 80: return launch_kv_t<80>(q, ldq, kv, ldkv, p, H, st);
    case 128: return launch_kv_t<128>(q, ldq, kv, ldkv, p, H, st);
    default: return launch_kv_t<64>(q, ldq, kv, ldkv, p, H, st);
  }
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
