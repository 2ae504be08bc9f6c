// RegionViT's region-to-local attention (reference regionvit.py:167-176), for sm_90a.
//   b200vit_attention_region_local   softmax attention inside every window of local tokens together with the window's
//                                    region token, under a learned relative-position bias between local tokens
//
// One buffer holds both token maps of the B images: the local tokens first, token (b, y, x) of the lh x lw map at row
// (b*lh + y)*lw + x, then the region tokens, token (b, i, j) of the rh x rw map at row B*lh*lw + (b*rh + i)*rw + j.
// Window (b, i, j) is the region token (b, i, j) and the wh x ww local tokens (i*wh + u, j*ww + v), wh = lh / rh and
// ww = lw / rw; its n = 1 + wh*ww tokens are numbered t = 0 (the region token) and t = 1 + u*ww + v.
//
// attention_region_local_kernel: one CTA = one warpgroup = one (window, head, 64-row query tile).  The tile's queries
// and the window's nkb = ceil(n / 64) key and value blocks (at most 4: n <= 256) are gathered with cp.async by their
// address map (tile64.cuh), tokens past n zero-filled without a read, so nothing is copied into window order.  Q and
// the K blocks land first; the V blocks load underneath the score pass.  Of the head's (2W-1)^2 bias values, the
// (2wh-1) x (2ww-1) offsets a window has are staged in shared memory, times log2 e.  Scores are S = scale Q K^T + bias
// per 64 x 64 block on wgmma, with bias 0 for every pair that involves the region token and keys past n dropped.
// With one key block the scores stay in registers; with more, a first pass finds each row's maximum over all blocks
// and a second pass recomputes each block (the same wgmma on the same operands, so the same bits) for exp2, the row
// sums and O += P V.  That keeps 32 score registers live instead of 32 per block.  Each result row goes back to its own row, local or region.
//
// Numerics: fp32 scores with scale * log2(e) folded into exp2 and the bias added in log2 units, probabilities exp2(s -
// row max) rounded to bf16 before P V, fp32 row sums and accumulation, one bf16 rounding of the output, as every
// attention kernel here.  Isolation: a CTA reads its window's rows only, and rows past n are zeros, never stale, so a
// NaN or Inf stays inside its window.
#include "tile64.cuh"
#include "host_util.h"

namespace {

using namespace b200;
using namespace b200::tile64;

constexpr int MAX_TOKENS = 256;   // one region token + wh*ww <= 255 local tokens: at most 4 key blocks

struct R2LParams {
  const __nv_bfloat16* qkv;
  const float* table;      // [H][(2W-1)^2]
  __nv_bfloat16* out;
  int lh, lw, rh, rw, wh, ww, W, I;  // I = H * dh
  long long local_rows;    // B * lh * lw: the first region row
  float scale_log2e;
};

template <int DH>
__global__ void __launch_bounds__(THREADS)
attention_region_local_kernel(const R2LParams p) {
  using S = Slabs<DH>;
  constexpr int N64 = S::N64, N16 = S::N16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int win = blockIdx.x, h = blockIdx.y, q0 = blockIdx.z * ROWS;
  const int nreg = p.rh * p.rw;
  const int b = win / nreg, ri = (win / p.rw) % p.rh, rj = win % p.rw;
  const int ww = p.ww, n = 1 + p.wh * ww, nkb = (n + ROWS - 1) / ROWS;
  const int tw = 2 * p.W - 1, bh = 2 * p.wh - 1, bw = 2 * ww - 1;   // the table's side, the window's offsets
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long ld = 3LL * p.I;
  float* tab = reinterpret_cast<float*>(smem + (1 + 2 * nkb) * S::OP);

  // window token t -> its row of qkv / out; -1 past the window (zero-filled without a read)
  auto row_of = [&](int t) -> long long {
    if (t >= n) return -1;
    if (t == 0) return p.local_rows + (long long)win;   // windows are numbered (b, i, j) as the region rows
    const int u = (t - 1) / ww, v = (t - 1) - ((t - 1) / ww) * ww;
    return ((long long)b * p.lh + ri * p.wh + u) * p.lw + rj * ww + v;
  };
  const uint32_t sq = smem_u32(smem), sk = sq + S::OP, sv = sq + (1 + nkb) * S::OP;
  load_block<DH>(sq, p.qkv, ld, h * DH, [&](int r) { return row_of(q0 + r); }, tid);
  for (int kb = 0; kb < nkb; ++kb)
    load_block<DH>(sk + kb * S::OP, p.qkv, ld, p.I + h * DH, [&](int r) { return row_of(kb * ROWS + r); }, tid);
  cp_async_commit();
  for (int kb = 0; kb < nkb; ++kb)
    load_block<DH>(sv + kb * S::OP, p.qkv, ld, 2 * p.I + h * DH, [&](int r) { return row_of(kb * ROWS + r); }, tid);
  cp_async_commit();
  // the bias of the offsets (du, dv) a wh x ww window has, at tab[(du + wh-1) + (dv + ww-1)*bh]
  const float* th = p.table + (long long)h * tw * tw + (p.W - p.wh) + (long long)(p.W - ww) * tw;
  for (int i = tid; i < bh * bw; i += THREADS) tab[i] = th[i % bh + (i / bh) * tw] * 1.4426950408889634f;
  cp_async_wait<1>();          // this thread's Q and K pieces have landed
  fence_proxy_async_smem();    // ... and are visible to wgmma
  __syncthreads();             // ... as are every other thread's, and the bias table

  // this thread's query tokens t = q0 + 16 warp + lane/4 + 8 rh as (u, v), -1 for the region token (rows past n: any
  // token, never stored)
  int qu[2], qv[2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    int t = q0 + warp * 16 + (lane >> 2) + 8 * rh;
    t = t < n ? t : 0;
    qu[rh] = t == 0 ? -1 : (t - 1) / ww;
    qv[rh] = t == 0 ? 0 : (t - 1) - qu[rh] * ww;
  }
  // s <- scale * S + bias of key block kb in log2 units, keys past n at -inf
  auto scores = [&](float (&s)[32], int kb) {
    wgmma_fence();
    qk_mma<DH>(s, sq, sk + kb * S::OP);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e1 = 0; e1 < 2; ++e1) {
        const int t = kb * ROWS + 8 * jj + 2 * (lane & 3) + e1;
        const bool ok = t < n;
        const int ku = t == 0 || !ok ? -1 : (t - 1) / ww, kv = ku < 0 ? 0 : (t - 1) - ku * ww;
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          const int e = 2 * rh + e1;
          const bool local = ku >= 0 && qu[rh] >= 0;
          const int idx = local ? (qu[rh] - ku + p.wh - 1) + (qv[rh] - kv + ww - 1) * bh : 0;
          const float bias = local ? tab[idx] : 0.f;
          s[4 * jj + e] = ok ? fmaf(s[4 * jj + e], p.scale_log2e, bias) : -INFINITY;
        }
      }
  };
  auto row_max = [&](const float (&s)[32], float (&mx)[2]) {
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 4; ++e) mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * jj + e]);
  };

  float s[32];
  float mx[2] = {-INFINITY, -INFINITY};
  for (int kb = 0; kb < nkb; ++kb) {   // with one key block, s keeps its scores for the pass below
    scores(s, kb);
    row_max(s, mx);
  }
  quad_max(mx);

  cp_async_wait<0>();          // the V blocks
  fence_proxy_async_smem();
  __syncthreads();

  float o[N64 > 0 ? N64 : 1][32], o16[N16 > 0 ? N16 : 1][8];
  zero_acc<DH>(o, o16);
  float l[2] = {0.f, 0.f};
  for (int kb = 0; kb < nkb; ++kb) {
    if (nkb > 1) scores(s, kb);
    tile_exp2(s, mx, l);
    wgmma_fence();
    pv_mma<DH>(o, o16, s, sv + kb * S::OP);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < N64; ++c) fence_regs(o[c]);
#pragma unroll
    for (int c = 0; c < N16; ++c) fence_regs(o16[c]);
  }
  quad_sum(l);

#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int t = q0 + warp * 16 + (lane >> 2) + 8 * rh;
    if (t >= n) continue;
    store_rows<DH>(o, o16, p.out + row_of(t) * p.I + h * DH + 2 * (lane & 3), rh, 1.0f / l[rh]);
  }
}

template <int DH>
int launch_region_local(const R2LParams& p, int windows, int H, int nkb, cudaStream_t stream) {
  // Q, nkb K and nkb V blocks, the window's bias values (at most 4 * 255); slack for 1024B alignment
  const int bytes = (1 + 2 * nkb) * Slabs<DH>::OP + (2 * p.wh - 1) * (2 * p.ww - 1) * 4 + 1024;
  auto kern = attention_region_local_kernel<DH>;
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3(windows, H, nkb), THREADS, bytes, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace

static inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

extern "C" int b200vit_attention_region_local(const void* qkv, void* out, const float* table, int B, int lh, int lw,
                                              int rh, int rw, int W, int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(qkv && out && table, "attention_region_local: null pointer");
  B200_CHECK_ARG(B > 0 && lh > 0 && lw > 0 && rh > 0 && rw > 0 && W > 0 && H > 0,
                 "attention_region_local: bad shape B=%d local %d x %d region %d x %d W=%d H=%d", B, lh, lw, rh, rw,
                 W, H);
  B200_CHECK_ARG(dh == 32, "attention_region_local: dim_head=%d (this kernel is built for 32)", dh);
  B200_CHECK_ARG(lh % rh == 0 && lw % rw == 0,
                 "attention_region_local: the %d x %d local map is not divisible by the %d x %d region map", lh, lw,
                 rh, rw);
  const int wh = lh / rh, ww = lw / rw;
  B200_CHECK_ARG(wh <= W && ww <= W,
                 "attention_region_local: a %d x %d window exceeds window_size=%d of the bias table", wh, ww, W);
  B200_CHECK_ARG((long long)wh * ww + 1 <= MAX_TOKENS,
                 "attention_region_local: a %d x %d window and its region token exceed %d tokens", wh, ww, MAX_TOKENS);
  B200_CHECK_ARG(aligned16(qkv) && aligned16(out) && aligned16(table),
                 "attention_region_local: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535, "attention_region_local: H=%d exceeds the grid", H);
  const long long windows = (long long)B * rh * rw;
  B200_CHECK_ARG(windows <= 0x7fffffffLL, "attention_region_local: %lld windows exceed the grid", windows);
  const long long local_rows = (long long)B * lh * lw;
  B200_CHECK_ARG(local_rows + windows <= 0x7fffffffLL, "attention_region_local: %lld rows exceed the row index",
                 local_rows + windows);
  R2LParams p{};
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv);
  p.table = table;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.lh = lh;
  p.lw = lw;
  p.rh = rh;
  p.rw = rw;
  p.wh = wh;
  p.ww = ww;
  p.W = W;
  p.I = H * dh;
  p.local_rows = local_rows;
  p.scale_log2e = scale * 1.4426950408889634f;
  const int nkb = (wh * ww + 1 + ROWS - 1) / ROWS;
  return launch_region_local<32>(p, (int)windows, H, nkb, reinterpret_cast<cudaStream_t>(stream));
}
