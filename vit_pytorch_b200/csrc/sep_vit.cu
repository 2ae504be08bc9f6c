// Kernels of SepViT's depthwise separable self-attention (reference sep_vit.py:65-206), for sm_90a.  The token map of
// a stage is kept channels-last: token (b, y, x) of a gh x gw map at row (b*gh + y)*gw + x; window (b, wy, wx) of
// the nwy x nwx grid of p x p windows is number (b*nwy + wy)*nwx + wx, the reference's '(b x y)' order.
//   b200vit_attention_window_token   softmax attention inside every window among its p*p tokens and one learned
//                                    window token (sep_vit.py:139-168)
//   b200vit_window_mix               per image and head, attention over the windows whose queries and keys come from
//                                    the window tokens and whose value for window j at position w is window j's
//                                    attention output at w (sep_vit.py:182-201)
// The LayerNorm + GELU of the window-token outputs (sep_vit.py:96-98) is b200vit_head_layernorm_gelu (rowops.cu).
//
// attention_window_token_kernel: one CTA = one warpgroup = one (window, head), the tile64.cuh operand blocks.  Row 0
// of each of Q, K and V is the head's slice of the window token's q | k | v (tok_qkv, the same for every window),
// rows 1 .. p*p the window's tokens gathered with cp.async by their map rows, rows past p*p + 1 zero-filled without a
// read.  S = Q K^T, the keys past p*p + 1 get -inf, a plain fp32 softmax (every key of a row is in the tile), O = P V.
// Rows 1 .. p*p go to their map rows of `out`, row 0 to row `window` of tok_out.
//
// window_mix_kernel: one CTA = one (image, head) and a slice of the p*p window positions.  Q and K are the head's
// interleaved columns of wqk for the image's nw windows (rows past nw zero-filled), S = Q K^T and the softmax once;
// then for each position w of the slice, V_w = the nw rows (window j, position w) of o, through a two-buffer cp.async
// ring (V_{w+1} loads while P V_w runs), O_w = P V_w to the rows (window i, position w) of out.
//
// Numerics of both: fp32 scores with scale * log2(e) folded into exp2, probabilities rounded to bf16 before P V, fp32
// accumulation and one bf16 rounding of the output, as every attention kernel here.
// Isolation: a tile never holds rows of two windows (attention_window_token) or two images (window_mix), and the rows
// past the valid ones are zeros, never stale, so a NaN or Inf stays inside its window, resp. its image and head.
#include "tile64.cuh"
#include "host_util.h"

namespace {

using namespace b200;
using namespace b200::tile64;

struct WinTokParams {
  const __nv_bfloat16* qkv;
  const __nv_bfloat16* tok_qkv;  // [3I]
  __nv_bfloat16* out;
  __nv_bfloat16* tok_out;        // [B*nw, I], or NULL
  int gh, gw, p, nwy, nwx, I;
  float scale_log2e;
};

template <int DH>
__global__ void __launch_bounds__(THREADS)
attention_window_token_kernel(const WinTokParams p) {
  using S = Slabs<DH>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int h = blockIdx.y, win = blockIdx.x;
  const int b = win / (p.nwy * p.nwx), wy = (win / p.nwx) % p.nwy, wx = win % p.nwx;
  const int w = p.p, n = w * w + 1;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long ld = 3LL * p.I;

  // tile row r = 1 + u*w + v -> its map row; row 0 (the window token) and rows past the window: -1, zero-filled
  auto row_of = [&](int r) -> long long {
    if (r == 0 || r >= n) return -1;
    const int t = r - 1, u = t / w, v = t - (t / w) * w;
    return ((long long)b * p.gh + wy * w + u) * p.gw + wx * w + v;
  };
  const uint32_t sq = smem_u32(smem), sk = sq + S::OP, sv = sq + 2 * S::OP;
  load_block<DH>(sq, p.qkv, ld, h * DH, row_of, tid);
  load_block<DH>(sk, p.qkv, ld, p.I + h * DH, row_of, tid);
  load_block<DH>(sv, p.qkv, ld, 2 * p.I + h * DH, row_of, tid);
  cp_async_commit();
  // row 0: piece c of each operand is the one load_block gave thread c (zero-filled); the same thread overwrites it
  // once its own cp.async group has landed
  constexpr int P = DH / 8;
  uint4 tok[3];
  if (tid < P) {
#pragma unroll
    for (int o = 0; o < 3; ++o)
      tok[o] = *reinterpret_cast<const uint4*>(p.tok_qkv + o * p.I + h * DH + 8 * tid);
  }
  cp_async_wait<0>();
  if (tid < P) {
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      const uint32_t a = piece_addr<DH>(sq + o * S::OP, 0, tid);
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(tok[o].x), "r"(tok[o].y), "r"(tok[o].z),
                   "r"(tok[o].w)
                   : "memory");
    }
  }
  fence_proxy_async_smem();    // the pieces are visible to wgmma
  __syncthreads();             // ... every thread's

  float s[32];
  wgmma_fence();
  qk_mma<DH>(s, sq, sk);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);
  float l[2];
  tile_softmax(s, l, n, p.scale_log2e, lane);

  float o[S::N64 > 0 ? S::N64 : 1][32], o16[S::N16 > 0 ? S::N16 : 1][8];
  zero_acc<DH>(o, o16);
  wgmma_fence();
  pv_mma<DH>(o, o16, s, sv);
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < S::N64; ++c) fence_regs(o[c]);
#pragma unroll
  for (int c = 0; c < S::N16; ++c) fence_regs(o16[c]);

#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int r = warp * 16 + (lane >> 2) + 8 * rh;
    if (r >= n) continue;
    __nv_bfloat16* dst;
    if (r == 0) {
      if (!p.tok_out) continue;
      dst = p.tok_out + (long long)win * p.I;
    } else {
      dst = p.out + row_of(r) * p.I;
    }
    store_rows<DH>(o, o16, dst + h * DH + 2 * (lane & 3), rh, 1.0f / l[rh]);
  }
}

template <int DH>
int launch_window_token(const WinTokParams& p, int windows, int H, cudaStream_t stream) {
  const int bytes = 3 * Slabs<DH>::OP + 1024;  // slack for 1024B alignment
  auto kern = attention_window_token_kernel<DH>;
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3(windows, H), THREADS, bytes, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------ window_mix
struct MixParams {
  const __nv_bfloat16* wqk;  // [B*nw, 2I], head h: q columns [2h dh, 2h dh + dh), k columns [2h dh + dh, 2(h+1) dh)
  const __nv_bfloat16* o;    // [B*gh*gw, I]
  __nv_bfloat16* out;        // [B*gh*gw, I]
  int H, gh, gw, p, nwy, nwx, I;
  int per;                   // window positions per CTA
  float scale_log2e;
};

template <int DH>
__global__ void __launch_bounds__(THREADS)
window_mix_kernel(const MixParams p) {
  using S = Slabs<DH>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int b = blockIdx.x / p.H, h = blockIdx.x % p.H;
  const int w = p.p, pp = w * w, nw = p.nwy * p.nwx;
  const int w0 = blockIdx.y * p.per, cnt = min(p.per, pp - w0);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // window j at window position q = u*w + v -> its map row; windows past nw: -1, zero-filled
  auto map_row = [&](int j, int q) -> long long {
    const int wy = j / p.nwx, wx = j - (j / p.nwx) * p.nwx, u = q / w, v = q - (q / w) * w;
    return ((long long)b * p.gh + wy * w + u) * p.gw + wx * w + v;
  };
  const uint32_t sq = smem_u32(smem), sk = sq + S::OP, sv0 = sq + 2 * S::OP;
  auto win_row = [&](int j) -> long long { return j < nw ? (long long)b * nw + j : -1; };
  load_block<DH>(sq, p.wqk, 2LL * p.I, 2 * h * DH, win_row, tid);
  load_block<DH>(sk, p.wqk, 2LL * p.I, 2 * h * DH + DH, win_row, tid);
  cp_async_commit();
  auto load_v = [&](int k) {
    const int q = w0 + k;
    load_block<DH>(sv0 + (k & 1) * S::OP, p.o, p.I, h * DH,
                   [&](int j) -> long long { return j < nw ? map_row(j, q) : -1; }, tid);
    cp_async_commit();
  };
  load_v(0);
  cp_async_wait<1>();          // Q and K have landed (V_0 may still be in flight)
  fence_proxy_async_smem();
  __syncthreads();

  float s[32];
  wgmma_fence();
  qk_mma<DH>(s, sq, sk);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);
  float l[2];
  tile_softmax(s, l, nw, p.scale_log2e, lane);
  const float inv[2] = {1.0f / l[0], 1.0f / l[1]};

  float o[S::N64 > 0 ? S::N64 : 1][32], o16[S::N16 > 0 ? S::N16 : 1][8];
  for (int k = 0; k < cnt; ++k) {
    if (k + 1 < cnt) {
      load_v(k + 1);           // into the buffer P V_{k-1} read, which every thread finished before the last barrier
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();           // V_k is complete, every thread's pieces
    zero_acc<DH>(o, o16);
    wgmma_fence();
    pv_mma<DH>(o, o16, s, sv0 + (k & 1) * S::OP);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < S::N64; ++c) fence_regs(o[c]);
#pragma unroll
    for (int c = 0; c < S::N16; ++c) fence_regs(o16[c]);
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      const int i = warp * 16 + (lane >> 2) + 8 * rh;
      if (i >= nw) continue;
      store_rows<DH>(o, o16, p.out + map_row(i, w0 + k) * p.I + h * DH + 2 * (lane & 3), rh, inv[rh]);
    }
    __syncthreads();           // every thread's P V_k is done before its buffer is refilled
  }
}

template <int DH>
int launch_mix(const MixParams& p, int B, int slices, cudaStream_t stream) {
  const int bytes = 4 * Slabs<DH>::OP + 1024;  // Q, K, two V buffers; slack for 1024B alignment
  auto kern = window_mix_kernel<DH>;
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3(B * p.H, slices), THREADS, bytes, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace

static inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

extern "C" int b200vit_attention_window_token(const void* qkv, const void* tok_qkv, void* out, void* tok_out, int B,
                                              int gh, int gw, int p, int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(qkv && tok_qkv && out, "attention_window_token: null pointer");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && p > 0 && H > 0,
                 "attention_window_token: bad shape B=%d h=%d w=%d p=%d H=%d", B, gh, gw, p, H);
  B200_CHECK_ARG(head_width_ok(dh),
                 "attention_window_token: dim_head=%d not supported by this build (32, 64, 80 or 128)", dh);
  B200_CHECK_ARG(p * p + 1 <= ROWS,
                 "attention_window_token: p=%d, a window of %d tokens and its window token must fit one %d-row tile",
                 p, p * p, ROWS);
  B200_CHECK_ARG(gh % p == 0 && gw % p == 0,
                 "attention_window_token: the %d x %d map is not divisible into %d x %d windows", gh, gw, p, p);
  B200_CHECK_ARG(aligned16(qkv) && aligned16(tok_qkv) && aligned16(out) && aligned16(tok_out),
                 "attention_window_token: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535, "attention_window_token: H=%d exceeds the grid", H);
  const long long windows = (long long)B * (gh / p) * (gw / p);
  B200_CHECK_ARG(windows <= 0x7fffffffLL, "attention_window_token: %lld windows exceed the grid", windows);
  WinTokParams q{};
  q.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv);
  q.tok_qkv = reinterpret_cast<const __nv_bfloat16*>(tok_qkv);
  q.out = reinterpret_cast<__nv_bfloat16*>(out);
  q.tok_out = reinterpret_cast<__nv_bfloat16*>(tok_out);
  q.gh = gh;
  q.gw = gw;
  q.p = p;
  q.nwy = gh / p;
  q.nwx = gw / p;
  q.I = H * dh;
  q.scale_log2e = scale * 1.4426950408889634f;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: return launch_window_token<32>(q, (int)windows, H, st);
    case 80: return launch_window_token<80>(q, (int)windows, H, st);
    case 128: return launch_window_token<128>(q, (int)windows, H, st);
    default: return launch_window_token<64>(q, (int)windows, H, st);
  }
}

extern "C" int b200vit_window_mix(const void* wqk, const void* o, void* out, int B, int gh, int gw, int p, int H,
                                  int dh, float scale, void* stream) {
  B200_CHECK_ARG(wqk && o && out, "window_mix: null pointer");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && p > 0 && H > 0, "window_mix: bad shape B=%d h=%d w=%d p=%d H=%d", B,
                 gh, gw, p, H);
  B200_CHECK_ARG(head_width_ok(dh), "window_mix: dim_head=%d not supported by this build (32, 64, 80 or 128)", dh);
  B200_CHECK_ARG(gh % p == 0 && gw % p == 0, "window_mix: the %d x %d map is not divisible into %d x %d windows", gh,
                 gw, p, p);
  const long long nw = (long long)(gh / p) * (gw / p);
  B200_CHECK_ARG(nw >= 2 && nw <= ROWS, "window_mix: %lld windows per map (2 to %d)", nw, ROWS);
  B200_CHECK_ARG(o != out, "window_mix: out must not be o (every output row reads the rows of all windows)");
  B200_CHECK_ARG(aligned16(wqk) && aligned16(o) && aligned16(out), "window_mix: pointers must be 16-byte aligned");
  B200_CHECK_ARG((long long)B * H <= 0x7fffffffLL, "window_mix: B*H=%lld exceeds the grid", (long long)B * H);
  MixParams q{};
  q.wqk = reinterpret_cast<const __nv_bfloat16*>(wqk);
  q.o = reinterpret_cast<const __nv_bfloat16*>(o);
  q.out = reinterpret_cast<__nv_bfloat16*>(out);
  q.H = H;
  q.gh = gh;
  q.gw = gw;
  q.p = p;
  q.nwy = gh / p;
  q.nwx = gw / p;
  q.I = H * dh;
  // at most 8 window positions per CTA, spread evenly over the slices (p = 7: 7 slices of 7)
  const int pp = p * p, slices_min = (pp + 7) / 8;
  q.per = (pp + slices_min - 1) / slices_min;
  const int slices = (pp + q.per - 1) / q.per;
  B200_CHECK_ARG(slices <= 65535, "window_mix: p=%d gives %d slices, beyond the grid", p, slices);
  q.scale_log2e = scale * 1.4426950408889634f;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: return launch_mix<32>(q, B, slices, st);
    case 80: return launch_mix<80>(q, B, slices, st);
    case 128: return launch_mix<128>(q, B, slices, st);
    default: return launch_mix<64>(q, B, slices, st);
  }
}
