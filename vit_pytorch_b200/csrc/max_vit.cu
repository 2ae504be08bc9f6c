// Kernels of MaxViT (reference max_vit.py), for sm_90a.  The token map of a stage is kept channels-last: x[B*h*w, C],
// token (b, y, x) at row (b*h + y)*w + x, whether the attention groups it into blocks or into dilated grids.
//   b200vit_attention_window_relpos   softmax attention inside w x w windows, block or grid partition, with a learned
//                                     relative-position bias (max_vit.py:121-206)
//   b200vit_mbconv_dwconv             depthwise 3 x 3 convolution, BatchNorm folded, GELU, and the per-image channel
//                                     sums squeeze-excitation averages (max_vit.py:106-109)
//   b200vit_se_pool / b200vit_se_scale  the squeeze-excitation mean and gate around its two GEMMs (max_vit.py:47-62)
//
// attention_window_relpos: one CTA = one warpgroup = one (window, head).  The window's w*w rows are gathered with
// cp.async into one 64-row tile (gather64.cuh), rows past w*w zero-filled without a read, so only the partition's
// address map differs between block and grid windows.  The head's (2w-1)^2 bias values (times log2 e) are staged in
// shared memory; each (query, key) index is formed from the local coordinates in registers.  S = Q K^T with wgmma, the
// bias added, keys past w*w masked to -inf, a plain fp32 softmax (every key of a row is in the tile), O = P V with
// wgmma.  One window per tile: for w = 7 a tile holds 49 of its 64 rows; packing windows is left undone.
//
// mbconv_dwconv: one thread = two adjacent channels of one image over a run of B200VIT_MBCONV_PART_ROWS output
// tokens; a warp reads 64 consecutive channels of a token per tap (128 B).  The thread sums its bf16-rounded outputs
// in token order and writes the sum to its own slot of `part`, which se_pool adds up in part order.
#include "gather64.cuh"
#include "host_util.h"

namespace {

using namespace b200;
using namespace b200::gather64;

struct RelposParams {
  const __nv_bfloat16* qkv;
  const float* table;      // [H][(2w-1)^2]
  __nv_bfloat16* out;
  int gh, gw, w, grid, I;  // I = H * dh
  int X, Y;                // windows along y and x
  float scale_log2e;
};

template <int DH>
__global__ void __launch_bounds__(PB_THREADS)
attention_window_relpos_kernel(const RelposParams p) {
  using S = PbSlabs<DH>;
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
  for (int i = tid; i < tw * tw; i += PB_THREADS) tab[i] = th[i] * 1.4426950408889634f;
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
  const int bytes = 3 * PbSlabs<DH>::OP + tw * tw * 4 + 1024;  // slack for 1024B alignment
  auto kern = attention_window_relpos_kernel<DH>;
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3(windows, H), PB_THREADS, bytes, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------ mbconv_dwconv
constexpr int DW_THREADS = 128;

__global__ void __launch_bounds__(DW_THREADS)
mbconv_dwconv_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w9, const float* __restrict__ bias,
                     __nv_bfloat16* __restrict__ y, float* __restrict__ part, int h, int w, int oh, int ow, int C,
                     int s, int P) {
  const int c = (blockIdx.x * DW_THREADS + threadIdx.x) * 2;
  if (c >= C) return;
  const int pi = blockIdx.y, b = blockIdx.z;
  const int n = oh * ow;
  const int t0 = pi * B200VIT_MBCONV_PART_ROWS;
  const int t1 = min(t0 + B200VIT_MBCONV_PART_ROWS, n);
  float2 wt[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) wt[k] = *reinterpret_cast<const float2*>(w9 + (long long)k * C + c);
  const float2 bb = *reinterpret_cast<const float2*>(bias + c);
  const __nv_bfloat16* xb = x + (long long)b * h * w * C + c;
  __nv_bfloat16* yb = y + (long long)b * n * C + c;
  float sum0 = 0.f, sum1 = 0.f;
  for (int t = t0; t < t1; ++t) {
    const int oy = t / ow, ox = t - (t / ow) * ow;
    float a0 = bb.x, a1 = bb.y;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = oy * s - 1 + ky;
      if (iy < 0 || iy >= h) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = ox * s - 1 + kx;
        if (ix < 0 || ix >= w) continue;
        const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(xb + ((long long)iy * w + ix) * C));
        a0 = fmaf(wt[3 * ky + kx].x, v.x, a0);
        a1 = fmaf(wt[3 * ky + kx].y, v.y, a1);
      }
    }
    gelu_erf2(a0, a1);
    const uint32_t pk = pack_bf16x2(a0, a1);
    *reinterpret_cast<uint32_t*>(yb + (long long)t * C) = pk;
    sum0 += __uint_as_float(pk << 16);
    sum1 += __uint_as_float(pk & 0xFFFF0000u);
  }
  *reinterpret_cast<float2*>(part + ((long long)b * P + pi) * C + c) = make_float2(sum0, sum1);
}

// ------------------------------------------------------------------------------------------------ se_pool / se_scale
__global__ void __launch_bounds__(256)
se_pool_kernel(const float* __restrict__ part, __nv_bfloat16* __restrict__ pooled, int P, int C, float inv_n) {
  const int c = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
  if (c >= C) return;
  const float* pp = part + (long long)b * P * C + c;
  float sum = 0.f;
  for (int i = 0; i < P; ++i) sum += pp[(long long)i * C];
  pooled[(long long)b * C + c] = __float2bfloat16_rn(sum * inv_n);
}

// one thread per 8 channels of one token
__global__ void __launch_bounds__(256)
se_scale_kernel(__nv_bfloat16* __restrict__ hbuf, const __nv_bfloat16* __restrict__ gate, long long total8, int n,
                int C) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= total8) return;
  const int C8 = C >> 3;
  const long long tok = i / C8;
  const int c = (int)(i - tok * C8) * 8;
  const long long b = tok / n;
  uint4* hp = reinterpret_cast<uint4*>(hbuf + tok * C + c);
  uint4 hv = *hp;
  const uint4 gv = *reinterpret_cast<const uint4*>(gate + b * C + c);
  uint32_t* hw = reinterpret_cast<uint32_t*>(&hv);
  const uint32_t* gw = reinterpret_cast<const uint32_t*>(&gv);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hw[k]));
    const float2 gf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&gw[k]));
    hw[k] = pack_bf16x2(hf.x * gf.x, hf.y * gf.y);
  }
  *hp = hv;
}

}  // namespace

static inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

extern "C" int b200vit_attention_window_relpos(const void* qkv, void* out, const float* table, int B, int gh, int gw,
                                               int w, int grid, int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(qkv && out && table, "attention_window_relpos: null pointer");
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && w > 0 && H > 0,
                 "attention_window_relpos: bad shape B=%d h=%d w=%d window=%d H=%d", B, gh, gw, w, H);
  B200_CHECK_ARG(head_width_ok(dh), "attention_window_relpos: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(w * w <= PB_ROWS, "attention_window_relpos: window=%d, %d tokens must fit one %d-row tile", w, w * w,
                 PB_ROWS);
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

extern "C" int b200vit_mbconv_dwconv(const void* x, int64_t M, const float* w9, const float* bias, void* y, float* part,
                                     int B, int h, int w, int C, int stride, void* stream) {
  B200_CHECK_ARG(x && w9 && bias && y && part, "mbconv_dwconv: null pointer");
  B200_CHECK_ARG(B > 0 && h > 0 && w > 0 && C > 0, "mbconv_dwconv: bad shape B=%d h=%d w=%d C=%d", B, h, w, C);
  B200_CHECK_ARG(stride == 1 || stride == 2, "mbconv_dwconv: stride=%d (1 or 2)", stride);
  B200_CHECK_ARG(M == (int64_t)B * h * w, "mbconv_dwconv: x has %lld rows, %lld expected", (long long)M,
                 (long long)B * h * w);
  B200_CHECK_ARG(C % 8 == 0, "mbconv_dwconv: C=%d must be a multiple of 8", C);
  B200_CHECK_ARG(x != y, "mbconv_dwconv: y must not be x (every token reads its neighbours)");
  B200_CHECK_ARG(aligned16(x) && aligned16(w9) && aligned16(bias) && aligned16(y) && aligned16(part),
                 "mbconv_dwconv: pointers must be 16-byte aligned");
  const int oh = (h + stride - 1) / stride, ow = (w + stride - 1) / stride;
  const long long P = ((long long)oh * ow + B200VIT_MBCONV_PART_ROWS - 1) / B200VIT_MBCONV_PART_ROWS;
  B200_CHECK_ARG(B <= 65535 && P <= 65535, "mbconv_dwconv: B=%d, %lld parts exceed the grid", B, P);
  const dim3 grid((C / 2 + DW_THREADS - 1) / DW_THREADS, (unsigned)P, B);
  mbconv_dwconv_kernel<<<grid, DW_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), w9, bias, reinterpret_cast<__nv_bfloat16*>(y), part, h, w, oh, ow, C,
      stride, (int)P);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_se_pool(const float* part, void* pooled, int B, int P, int C, float inv_n, void* stream) {
  B200_CHECK_ARG(part && pooled, "se_pool: null pointer");
  B200_CHECK_ARG(B > 0 && P > 0 && C > 0, "se_pool: bad shape B=%d P=%d C=%d", B, P, C);
  B200_CHECK_ARG(C % 8 == 0, "se_pool: C=%d must be a multiple of 8", C);
  B200_CHECK_ARG(aligned16(part) && aligned16(pooled), "se_pool: pointers must be 16-byte aligned");
  B200_CHECK_ARG(B <= 65535, "se_pool: B=%d exceeds the grid", B);
  se_pool_kernel<<<dim3((C + 255) / 256, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      part, reinterpret_cast<__nv_bfloat16*>(pooled), P, C, inv_n);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_se_scale(void* h, const void* gate, int B, int n, int C, void* stream) {
  B200_CHECK_ARG(h && gate, "se_scale: null pointer");
  B200_CHECK_ARG(B > 0 && n > 0 && C > 0, "se_scale: bad shape B=%d n=%d C=%d", B, n, C);
  B200_CHECK_ARG(C % 8 == 0, "se_scale: C=%d must be a multiple of 8", C);
  B200_CHECK_ARG(aligned16(h) && aligned16(gate), "se_scale: pointers must be 16-byte aligned");
  const long long total8 = (long long)B * n * (C / 8);
  B200_CHECK_ARG((total8 + 255) / 256 <= 0x7fffffffLL, "se_scale: %lld elements exceed the grid", total8 * 8);
  se_scale_kernel<<<(unsigned)((total8 + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<__nv_bfloat16*>(h), reinterpret_cast<const __nv_bfloat16*>(gate), total8, n, C);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
