// Softmax attention over token groups small enough that every key of a query fits one 64-row wgmma tile (sm_90a):
//   b200vit_attention_axial           ViViT's attention along the time axis (reference vivit.py:144-150) and the
//                                     masked temporal transformer (vivit.py:268), with an optional per-sequence
//                                     key mask
//   b200vit_attention_window          Twins-SVT's attention inside non-overlapping p x p windows (twins_svt.py:85-120)
//   b200vit_attention_window_relpos   MaxViT's block or grid window attention with a learned relative-position bias
//                                     (max_vit.py:121-206)
//
// The tile scheme.  One CTA = one warpgroup = one 64-row tile of one head (tile64.cuh operand slabs, dh = 32, 64, 80 or
// 128) that holds whole softmax groups of one image.  S = Q K^T (64 x 64) with wgmma; keys outside the query's group
// get the score -inf in registers; a plain fp32 softmax, since every key of a row is in the tile; O = P V with wgmma,
// P (bf16) taken from registers as the A operand and V read as the transposed (MN-major) B operand.
//
// attention_tile_kernel (axial and window).  Both read B token maps of gw x gh tokens, token (b, y, x) at row
// (b*gh + y)*gw + x of qkv[., 3*H*dh] and of out, cut into windows wx tokens wide and wy tall; a window is one group.
// A tile holds spx x spy whole windows: a box bw = wx spx tokens wide and bh = wy spy tall at (tx bw, ty bh), tile
// row r = iy * bw + ix.  Thread 0 loads Q, K and V with one TMA box per slab over the 4-D view (column, x, y, b) of
// qkv; tokens outside the map are zero-filled, tile rows past the box are zeroed by the CTA first.
//   window: wx = wy = p, as many windows per tile as fit, along x first.
//   axial:  the map of batch element b is G wide (x = position p) and L tall (y = time j), wx = 1, wy = L,
//           spx = min(G, 64 / L), spy = 1: the tile holds spx whole sequences, row r = j * spx + ip.  An optional key
//           mask [B][L] (1 = keep) drops keys.
// A key is kept for a query when it lies in the query's window, in the box and the map, and is not masked.  Whether a
// query row has a kept key is decided from these indices and the mask, never from the scores.  A row without one gets
// 0 (zero_masked_rows, scaled_dot_product_attention's result) or the mean of its window's values (masked_fill(
// -finfo.max) before the softmax, vivit.py:91-94).  Every other row is exp2(s - max) over its kept keys, so a row
// whose kept scores are all NaN or all -inf is NaN, as the reference's softmax is.
//
// attention_window_relpos_kernel.  One (window, head) per tile: the window's w*w rows are gathered with cp.async
// (tile64.cuh), rows past w*w zero-filled without a read, so only the partition's address map differs between block
// and grid windows.  The head's (2w-1)^2 bias values (times log2 e) are staged in shared memory; each (query, key)
// index is formed from the local coordinates in registers and the bias added to the scaled score.  Every stored row
// has w*w kept keys.  One window per tile: for w = 7 a tile holds 49 of its 64 rows; packing windows is left undone.
// It keeps a kernel body of its own: folded into attention_tile_kernel as a second loader, the bias lookup under the
// per-row key mask costs it 20 or more registers at dh = 32, MaxViT's head width.
//
// Isolation.  A tile never holds two images: O = P V meets every V row of the tile, and a zero probability times a
// NaN or Inf value would carry one image's non-finite input into another's output.  For the same reason rows past the
// box or the window are zero, never stale.  Windows that share a tile meet each other's V rows with probability
// exactly 0, so a finite change in one window leaves the others bit-identical; a NaN or Inf stays within its image,
// and within its window when the window has a tile of its own.
#include "tile64.cuh"
#include "host_util.h"

namespace {

using namespace b200;
using namespace b200::tile64;

struct TileParams {
  __nv_bfloat16* out;
  const uint8_t* key_mask;  // NULL, or [B][gh]: key (b, y, x) is dropped where key_mask[b*gh + y] == 0
  int B, gh, gw, I;         // I = H * dh
  int wx, wy;               // the window, in tokens
  int spx, spy;             // windows per tile along x and y
  int tiles_x, tiles_y;     // tiles per image along x and y
  float scale_log2e;
  int zero_masked_rows;
};

template <int DH>
__global__ void __launch_bounds__(THREADS)
attention_tile_kernel(const __grid_constant__ CUtensorMap tm64, const __grid_constant__ CUtensorMap tm16,
                      const TileParams p) {
  using S = Slabs<DH>;
  constexpr int N64 = S::N64, N16 = S::N16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 3 * S::OP);

  const int h = blockIdx.y;
  const int tx = blockIdx.x % p.tiles_x, ty = (blockIdx.x / p.tiles_x) % p.tiles_y;
  const int b0 = blockIdx.x / (p.tiles_x * p.tiles_y);
  const int bw = p.wx * p.spx, bh = p.wy * p.spy;  // the box, in tokens
  const int x0 = tx * bw, y0 = ty * bh;
  const int rows = bw * bh;                         // <= 64
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // rows beyond the box: their keys are never kept, but V meets a zero probability in O = P V and must be finite
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int o = 0; o < 3; ++o) {
#pragma unroll
    for (int c = 0; c < N64; ++c) {
      uint4* sl = reinterpret_cast<uint4*>(smem + o * S::OP + c * S::S64);
      for (int i = rows * 8 + tid; i < ROWS * 8; i += THREADS) sl[i] = z;
    }
#pragma unroll
    for (int c = 0; c < N16; ++c) {
      uint4* sl = reinterpret_cast<uint4*>(smem + o * S::OP + N64 * S::S64 + c * S::S16);
      for (int i = rows * 2 + tid; i < ROWS * 2; i += THREADS) sl[i] = z;
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
  // the window of each within the tile; a key outside the box or the map is -1, a masked key its window + MASKED
  constexpr int MASKED = 128;  // above any window index of a 64-row tile
  int rwin[2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int r = warp * 16 + (lane >> 2) + 8 * rh;
    rwin[rh] = ((r / bw) / p.wy) * p.spx + (r % bw) / p.wx;
  }
  int cwin[16];
#pragma unroll
  for (int ci = 0; ci < 16; ++ci) {
    const int c = 8 * (ci >> 1) + 2 * (lane & 3) + (ci & 1);
    const int iy = c / bw, ix = c % bw;
    cwin[ci] = (c < rows && x0 + ix < p.gw && y0 + iy < p.gh) ? (iy / p.wy) * p.spx + ix / p.wx : -1;
    if (cwin[ci] >= 0 && p.key_mask && !p.key_mask[(long long)b0 * p.gh + y0 + iy]) cwin[ci] += MASKED;
  }

  mbar_wait(bar, 0);

  float s[32];
  const uint32_t sq = smem_u32(smem), sk = sq + S::OP, sv = sq + 2 * S::OP;
  wgmma_fence();
  qk_mma<DH>(s, sq, sk);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);

  // plain softmax in log2 units; s[4 jj + e]: row half rh = e >> 1, key column index ci = 2 jj + (e & 1).  A key is
  // kept when it is in the query's window, in the map and not masked; has, bit rh: row rh keeps a key in some lane of
  // its quad, decided from these indices alone
  float mx[2] = {-INFINITY, -INFINITY};
  uint32_t has = 0;
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int ci = 2 * jj + (e & 1), rh = e >> 1;
      const bool ok = cwin[ci] == rwin[rh];
      s[4 * jj + e] = ok ? s[4 * jj + e] * p.scale_log2e : -INFINITY;
      mx[rh] = fmaxf(mx[rh], s[4 * jj + e]);
      has |= (ok ? 1u : 0u) << rh;
    }
  has |= __shfl_xor_sync(0xffffffffu, has, 1);
  has |= __shfl_xor_sync(0xffffffffu, has, 2);
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
      const int ci = 2 * jj + (e & 1), rh = e >> 1;
      float v;
      // a row with a kept key: the others have the score -inf, so probability 0 beside a finite maximum
      if ((has >> rh) & 1u) v = fast_ex2(s[4 * jj + e] - mx[rh]);
      else v = (!p.zero_masked_rows && (cwin[ci] & ~MASKED) == rwin[rh]) ? 1.f : 0.f;  // none: 0, or its window's mean
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
// swizzle) by bw x bh x 1 tokens.  A kind the head does not use gets a copy of the other (never read).
template <int DH>
int launch_tile_t(const void* qkv, const TileParams& p, int H, int tiles, cudaStream_t stream) {
  using S = Slabs<DH>;
  CUtensorMap tm[2];
  const uint64_t ld = (uint64_t)3 * p.I;
  const uint64_t dims[4] = {ld, (uint64_t)p.gw, (uint64_t)p.gh, (uint64_t)p.B};
  const uint64_t strides[3] = {ld * 2, ld * 2 * p.gw, ld * 2 * p.gw * p.gh};
  const uint32_t bw = (uint32_t)(p.wx * p.spx), bh = (uint32_t)(p.wy * p.spy);
  const uint32_t box64[4] = {64, bw, bh, 1};
  const uint32_t box16[4] = {16, bw, bh, 1};
  int rc = 0;
  if (S::N64) rc = encode_tmap_bf16(&tm[0], qkv, 4, dims, strides, box64);
  if (!rc && S::N16) rc = encode_tmap_bf16_sw(&tm[1], qkv, 4, dims, strides, box16, 32);
  if (rc) return rc;
  if (!S::N16) tm[1] = tm[0];
  if (!S::N64) tm[0] = tm[1];
  auto kern = attention_tile_kernel<DH>;
  const int bytes = 3 * S::OP + 8 + 1024;  // barrier; slack for 1024B alignment
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3(tiles, H), THREADS, bytes, stream>>>(tm[0], tm[1], p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int launch_tile(const void* qkv, const TileParams& p, int H, int dh, int tiles, cudaStream_t st) {
  switch (dh) {
    case 32: return launch_tile_t<32>(qkv, p, H, tiles, st);
    case 80: return launch_tile_t<80>(qkv, p, H, tiles, st);
    case 128: return launch_tile_t<128>(qkv, p, H, tiles, st);
    default: return launch_tile_t<64>(qkv, p, H, tiles, st);
  }
}

// ------------------------------------------------------------------------------------------------ window_relpos
struct RelposParams {
  const __nv_bfloat16* qkv;
  const float* table;      // [H][(2w-1)^2]
  __nv_bfloat16* out;
  int gh, gw, w, grid, I;  // I = H * dh
  int X, Y;                // windows along y and x
  float scale_log2e;
};

template <int DH>
__global__ void __launch_bounds__(THREADS)
attention_window_relpos_kernel(const RelposParams p) {
  using S = Slabs<DH>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* tab = reinterpret_cast<float*>(smem + 3 * S::OP);

  const int h = blockIdx.y, win = blockIdx.x;
  const int b = win / (p.X * p.Y), wi = (win / p.Y) % p.X, wj = win % p.Y;
  const int w = p.w, n = w * w, tw = 2 * w - 1;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long ld = 3LL * p.I;

  // local token r = u*w + v of the window -> its row of the map, -1 past the window
  auto row_of = [&](int r) -> long long {
    if (r >= n) return -1;
    const int u = r / w, v = r - (r / w) * w;
    const int y = p.grid ? u * p.X + wi : wi * w + u;
    const int x = p.grid ? v * p.Y + wj : wj * w + v;
    return ((long long)b * p.gh + y) * p.gw + x;
  };
  const uint32_t sq = smem_u32(smem), sk = sq + S::OP, sv = sq + 2 * S::OP;
  load_block<DH>(sq, p.qkv, ld, h * DH, row_of, tid);
  load_block<DH>(sk, p.qkv, ld, p.I + h * DH, row_of, tid);
  load_block<DH>(sv, p.qkv, ld, 2 * p.I + h * DH, row_of, tid);
  cp_async_commit();
  const float* th = p.table + (long long)h * tw * tw;
  for (int i = tid; i < tw * tw; i += THREADS) tab[i] = th[i] * 1.4426950408889634f;
  cp_async_wait<0>();          // this thread's pieces have landed
  fence_proxy_async_smem();    // ... and are visible to wgmma
  __syncthreads();             // ... as are every other thread's, and the bias table

  float s[32];
  wgmma_fence();
  qk_mma<DH>(s, sq, sk);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);

  // this thread's rows r = 16 warp + lane/4 + 8 rh (rows past the window: any valid coordinates, never stored) and
  // key columns c = 8 jj + 2 (lane % 4) + e1
  int qu[2], qv[2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    int r = warp * 16 + (lane >> 2) + 8 * rh;
    r = r < n ? r : 0;
    qu[rh] = r / w;
    qv[rh] = r - qu[rh] * w;
  }
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e1 = 0; e1 < 2; ++e1) {
      const int c = 8 * jj + 2 * (lane & 3) + e1;
      const bool ok = c < n;
      const int cc = ok ? c : 0;
      const int ku = cc / w, kv = cc - (cc / w) * w;
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        const int e = 2 * rh + e1;
        const int idx = (qu[rh] - ku + w - 1) * tw + (qv[rh] - kv + w - 1);
        s[4 * jj + e] = ok ? fmaf(s[4 * jj + e], p.scale_log2e, tab[idx]) : -INFINITY;
        mx[rh] = fmaxf(mx[rh], s[4 * jj + e]);
      }
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
      const float v = fast_ex2(s[4 * jj + e] - mx[rh]);
      s[4 * jj + e] = v;
      l[rh] += v;
    }
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 1);
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 2);
  }

  constexpr int N64 = S::N64, N16 = S::N16;
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
    if (r >= n) continue;
    const float inv = 1.0f / l[rh];
    __nv_bfloat16* op = p.out + row_of(r) * p.I + h * DH + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < N64; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(op + 64 * c + jj * 8) =
            pack_bf16x2(o[c][4 * jj + 2 * rh] * inv, o[c][4 * jj + 2 * rh + 1] * inv);
#pragma unroll
    for (int c = 0; c < N16; ++c)
#pragma unroll
      for (int jj = 0; jj < 2; ++jj)
        *reinterpret_cast<uint32_t*>(op + 64 * N64 + 16 * c + jj * 8) =
            pack_bf16x2(o16[c][4 * jj + 2 * rh] * inv, o16[c][4 * jj + 2 * rh + 1] * inv);
  }
}

template <int DH>
int launch_relpos(const RelposParams& p, int windows, int H, cudaStream_t stream) {
  const int tw = 2 * p.w - 1;
  const int bytes = 3 * Slabs<DH>::OP + tw * tw * 4 + 1024;  // slack for 1024B alignment
  auto kern = attention_window_relpos_kernel<DH>;
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3(windows, H), THREADS, bytes, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}


}  // namespace

static inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

extern "C" int b200vit_attention_axial(const void* qkv, void* out, const uint8_t* key_mask, int B, int L, int G, int H,
                                       int dh, float scale, int zero_masked_rows, void* stream) {
  B200_CHECK_ARG(qkv && out, "attention_axial: null pointer");
  B200_CHECK_ARG(B > 0 && L > 0 && G > 0 && H > 0, "attention_axial: bad shape B=%d L=%d G=%d H=%d", B, L, G, H);
  B200_CHECK_ARG(head_width_ok(dh), "attention_axial: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(L <= ROWS, "attention_axial: L=%d > %d (a sequence must fit one 64-row tile)", L, ROWS);
  B200_CHECK_ARG(aligned16(qkv) && aligned16(out), "attention_axial: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535, "attention_axial: H=%d exceeds the grid", H);
  TileParams q{};
  q.out = reinterpret_cast<__nv_bfloat16*>(out);
  q.key_mask = key_mask;
  q.B = B;
  q.gh = L;
  q.gw = G;
  q.I = H * dh;
  q.wx = 1;
  q.wy = L;
  q.spx = G < ROWS / L ? G : ROWS / L;
  q.spy = 1;
  q.tiles_x = (G + q.spx - 1) / q.spx;
  q.tiles_y = 1;
  const long long tiles = (long long)q.tiles_x * B;
  B200_CHECK_ARG(tiles <= 0x7fffffffLL, "attention_axial: %lld tiles exceed the grid", tiles);
  q.scale_log2e = scale * 1.4426950408889634f;
  q.zero_masked_rows = zero_masked_rows != 0;
  return launch_tile(qkv, q, H, dh, (int)tiles, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b200vit_attention_window(const void* qkv, void* out, int B, int gh, int gw, int p, int H, int dh,
                                        float scale, void* stream) {
  B200_CHECK_ARG(qkv && out, "attention_window: null pointer");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && p > 0 && H > 0, "attention_window: bad shape B=%d h=%d w=%d p=%d H=%d", B,
                 gh, gw, p, H);
  B200_CHECK_ARG(head_width_ok(dh), "attention_window: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(p * p <= ROWS, "attention_window: p=%d, a window of %d tokens must fit one %d-row tile", p, p * p,
                 ROWS);
  B200_CHECK_ARG(gh % p == 0 && gw % p == 0, "attention_window: the %d x %d grid is not divisible into %d x %d windows",
                 gh, gw, p, p);
  B200_CHECK_ARG(aligned16(qkv) && aligned16(out), "attention_window: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535, "attention_window: H=%d exceeds the grid", H);
  TileParams q{};
  q.out = reinterpret_cast<__nv_bfloat16*>(out);
  q.B = B;
  q.gh = gh;
  q.gw = gw;
  q.wx = q.wy = p;
  q.I = H * dh;
  const int fit = ROWS / (p * p), wx = gw / p, wy = gh / p;
  q.spx = wx < fit ? wx : fit;
  q.spy = wy < fit / q.spx ? wy : fit / q.spx;
  q.tiles_x = (wx + q.spx - 1) / q.spx;
  q.tiles_y = (wy + q.spy - 1) / q.spy;
  const long long tiles = (long long)q.tiles_x * q.tiles_y * B;
  B200_CHECK_ARG(tiles <= 0x7fffffffLL, "attention_window: %lld tiles exceed the grid", tiles);
  q.scale_log2e = scale * 1.4426950408889634f;
  q.zero_masked_rows = 1;
  return launch_tile(qkv, q, H, dh, (int)tiles, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b200vit_attention_window_relpos(const void* qkv, void* out, const float* table, int B, int gh, int gw,
                                               int w, int grid, int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(qkv && out && table, "attention_window_relpos: null pointer");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && w > 0 && H > 0,
                 "attention_window_relpos: bad shape B=%d h=%d w=%d window=%d H=%d", B, gh, gw, w, H);
  B200_CHECK_ARG(head_width_ok(dh), "attention_window_relpos: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(w * w <= ROWS, "attention_window_relpos: window=%d, %d tokens must fit one %d-row tile", w, w * w,
                 ROWS);
  B200_CHECK_ARG(gh % w == 0 && gw % w == 0,
                 "attention_window_relpos: the %d x %d map is not divisible into %d x %d windows", gh, gw, w, w);
  B200_CHECK_ARG(grid == 0 || grid == 1, "attention_window_relpos: grid=%d (0 block, 1 grid)", grid);
  B200_CHECK_ARG(aligned16(qkv) && aligned16(out) && aligned16(table),
                 "attention_window_relpos: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535, "attention_window_relpos: H=%d exceeds the grid", H);
  const long long windows = (long long)B * (gh / w) * (gw / w);
  B200_CHECK_ARG(windows <= 0x7fffffffLL, "attention_window_relpos: %lld windows exceed the grid", windows);
  RelposParams p{};
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv);
  p.table = table;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.gh = gh;
  p.gw = gw;
  p.w = w;
  p.grid = grid;
  p.I = H * dh;
  p.X = gh / w;
  p.Y = gw / w;
  p.scale_log2e = scale * 1.4426950408889634f;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: return launch_relpos<32>(p, (int)windows, H, st);
    case 80: return launch_relpos<80>(p, (int)windows, H, st);
    case 128: return launch_relpos<128>(p, (int)windows, H, st);
    default: return launch_relpos<64>(p, (int)windows, H, st);
  }
}
