// The two operations of PiT (reference pit.py) that no other kernel covers.
//
// b200vit_unfold_patches: nn.Unfold(kernel_size=p, stride=s) + Rearrange('b c n -> b n c') (pit.py:140-147) as bit
//   copies into the A operand of the patch GEMM.  Patches overlap when s < p (PiT uses s = p / 2: every pixel lands in
//   up to four patches), so one CTA per (image, patch row, chunk of patch columns) stages the image rows that patch row
//   covers in shared memory, channel group by channel group, and writes every patch of the chunk from there: each pixel
//   is read from global memory once per patch row that covers it, not once per patch.  A gather, not TMA: a half-patch
//   stride in bytes (7 x 2 = 14 at p = 14) breaks TMA's 16-byte global-stride rule.
//
// b200vit_pit_pool: the token part of Pool (pit.py:98-113) up to the 1 x 1 convolution, whose GEMM follows: the
//   depthwise 3 x 3, stride 2, pad 1 convolution with channel multiplier 2 over the h x w token grid of the fp32
//   residual stream, plus a bf16 copy of every cls row (the A operand of cls_ff).  One CTA per (image, band of output
//   rows) stages the band's input rows plus a one-row halo, CH channels at a time, as lpi_kernel does; each thread owns
//   one input channel c and computes its two output channels 2c and 2c + 1.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

// img [B, C, H, W] bf16; out row b*oh*ow + r*ow + q, column (ch*p + i)*p + j = img[b, ch, r*s + i, q*s + j].
// CTA (b*oh + r, chunk): patch columns q0 .. q0 + nq - 1, image columns x0 = q0*s .. x0 + span - 1.
__global__ void __launch_bounds__(256)
unfold_kernel(const __nv_bfloat16* __restrict__ img, __nv_bfloat16* __restrict__ out, long long ldo, int C, int H,
              int W, int p, int s, int oh, int ow, int NQ, int CC) {
  extern __shared__ __nv_bfloat16 unfold_smem[];   // [cc][p][span]
  const int b = blockIdx.x / oh, r = blockIdx.x % oh;
  const int q0 = blockIdx.y * NQ;
  const int nq = ow - q0 < NQ ? ow - q0 : NQ;
  const int span = (nq - 1) * s + p, x0 = q0 * s, pp = p * p;
  const long long row0 = ((long long)b * oh + r) * ow + q0;
  const __nv_bfloat16* src = img + (long long)b * C * H * W + (long long)(r * s) * W + x0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  for (int c0 = 0; c0 < C; c0 += CC) {
    const int cc = C - c0 < CC ? C - c0 : CC;
    // one warp per staged image row (c, i), its lanes along the row
    for (int ri = warp; ri < cc * p; ri += warps) {
      const int c = ri / p, i = ri - c * p;
      const __nv_bfloat16* srow = src + (long long)(c0 + c) * H * W + (long long)i * W;
      for (int x = lane; x < span; x += 32) unfold_smem[ri * span + x] = srow[x];
    }
    __syncthreads();
    // column k of the channel group (c0*pp + k of every patch row) comes from the same staged element for every
    // patch, shifted by s per patch: its position is worked out once and the patches of the chunk are walked
    const int seg = cc * pp;
    for (int k = threadIdx.x; k < seg; k += blockDim.x) {
      const int c = k / pp, rem = k - c * pp, i = rem / p, j = rem - i * p;
      const __nv_bfloat16* from = unfold_smem + (c * p + i) * span + j;
      __nv_bfloat16* to = out + row0 * ldo + (long long)c0 * pp + k;
      for (int q = 0; q < nq; ++q) to[q * ldo] = from[q * s];
    }
    __syncthreads();
  }
  const int K = C * pp, pad = (int)(ldo - K);
  const __nv_bfloat16 zero = __float2bfloat16_rn(0.f);
  for (int k = threadIdx.x; k < pad; k += blockDim.x)
    for (int q = 0; q < nq; ++q) out[(row0 + q) * ldo + K + k] = zero;
}

// x fp32 [B*(1 + h*w), D], token t of image b at row b*(1 + h*w) + 1 + t.  w9 fp32 [9][2D] (tap dy*3 + dx major,
// output channel minor), b2 fp32 [2D].  a: row b*(1 + oh*ow) + 1 + t holds output token t (2D columns), row
// b*(1 + oh*ow) is the cls slot, zero filled.  cls: row b = bf16 copy of x's cls row of image b.
template <int CH>
__global__ void __launch_bounds__(256)
pit_pool_kernel(const float* __restrict__ x, const float* __restrict__ w9, const float* __restrict__ b2,
                __nv_bfloat16* __restrict__ a, long long lda, __nv_bfloat16* __restrict__ cls, long long ldc, int h,
                int w, int D, int RB) {
  constexpr int PL = 256 / CH;                  // position lanes
  const int oh = (h + 1) / 2, ow = (w + 1) / 2;
  const int WP = w + 2;                         // padded row: columns -1 .. w
  const int bands = (oh + RB - 1) / RB;
  const int b = blockIdx.x / bands, o0 = (blockIdx.x % bands) * RB;
  const int rb = oh - o0 < RB ? oh - o0 : RB;   // output rows of this CTA
  const int zrows = 2 * rb + 1;                 // input rows 2*o0 - 1 .. 2*(o0 + rb - 1) + 1
  extern __shared__ float4 pool_smem4[];
  float* zs = reinterpret_cast<float*>(pool_smem4);   // [zrows][WP][CH]
  const int tid = threadIdx.x, ch = tid % CH, pl = tid / CH;
  const float* xi = x + ((long long)b * (1 + h * w) + 1) * D;                 // token 0 of image b
  __nv_bfloat16* ai = a + ((long long)b * (1 + oh * ow) + 1) * lda;            // output token 0 of image b
  if (o0 == 0) {
    const __nv_bfloat16 zero = __float2bfloat16_rn(0.f);
    for (int c = tid; c < 2 * D; c += 256) ai[c - lda] = zero;
    for (int c = tid; c < D; c += 256) cls[(long long)b * ldc + c] = __float2bfloat16_rn(xi[c - D]);
  }
  for (int c0 = 0; c0 < D; c0 += CH) {
    const int c = c0 + ch;
    float w0[9], w1[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const float2 v = *reinterpret_cast<const float2*>(w9 + (long long)i * 2 * D + 2 * c);
      w0[i] = v.x;
      w1[i] = v.y;
    }
    const float2 bias = *reinterpret_cast<const float2*>(b2 + 2 * c);
    for (int zr = 0; zr < zrows; ++zr) {
      const int rr = 2 * o0 - 1 + zr;
      for (int pc = pl; pc < WP; pc += PL) {
        const int col = pc - 1;
        float v = 0.f;
        if (rr >= 0 && rr < h && col >= 0 && col < w) v = xi[((long long)rr * w + col) * D + c];
        zs[(zr * WP + pc) * CH + ch] = v;
      }
    }
    __syncthreads();
    for (int orow = 0; orow < rb; ++orow) {
      for (int ocol = pl; ocol < ow; ocol += PL) {
        float acc0 = 0.f, acc1 = 0.f;
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
          for (int dx = 0; dx < 3; ++dx) {
            const float v = zs[((2 * orow + dy) * WP + 2 * ocol + dx) * CH + ch];
            acc0 = fmaf(w0[dy * 3 + dx], v, acc0);
            acc1 = fmaf(w1[dy * 3 + dx], v, acc1);
          }
        const long long t = (long long)(o0 + orow) * ow + ocol;
        *reinterpret_cast<__nv_bfloat162*>(ai + t * lda + 2 * c) = __floats2bfloat162_rn(acc0 + bias.x, acc1 + bias.y);
      }
    }
    __syncthreads();
  }
}

// (output rows per CTA, channel chunk) whose staged input rows fit in 48 KB of shared memory: the widest chunk that
// divides D, with up to 4 output rows per CTA (chunk 0: none fits, even one output row per CTA)
static int pool_tiling(int h, int w, int D, int* rows, size_t* smem) {
  const int oh = (h + 1) / 2;
  for (int rb = oh < 4 ? oh : 4;; rb = 1) {
    for (int ch = 32; ch >= 8; ch /= 2) {
      const size_t s = (size_t)(2 * rb + 1) * (size_t)(w + 2) * ch * sizeof(float);
      if (D % ch == 0 && s <= 48 * 1024) {
        *rows = rb;
        *smem = s;
        return ch;
      }
    }
    if (rb == 1) return 0;
  }
}

template <int CH>
static int launch_pool(int grid, size_t smem, cudaStream_t st, const float* x, const float* w9, const float* b2,
                       void* a, long long lda, void* cls, long long ldc, int h, int w, int D, int rb) {
  pit_pool_kernel<CH><<<grid, 256, smem, st>>>(x, w9, b2, reinterpret_cast<__nv_bfloat16*>(a), lda,
                                               reinterpret_cast<__nv_bfloat16*>(cls), ldc, h, w, D, rb);
  return 0;
}

}  // namespace b200

using namespace b200;

static constexpr int kUnfoldSmem = 48 * 1024;

extern "C" int b200vit_unfold_patches(const void* img, void* out_bf16, int64_t ldo, int B, int C, int H, int W, int p,
                                      int s, void* stream) {
  B200_CHECK_ARG(img && out_bf16, "unfold_patches: null pointer");
  B200_CHECK_ARG(B > 0 && C > 0 && p >= 2 && s >= 1 && H >= p && W >= p,
                 "unfold_patches: bad shape B=%d C=%d H=%d W=%d p=%d s=%d (p >= 2, s >= 1, H and W >= p)", B, C, H, W,
                 p, s);
  const int oh = (H - p) / s + 1, ow = (W - p) / s + 1;
  const long long K = (long long)C * p * p, rows = (long long)B * oh * ow;
  B200_CHECK_ARG(ldo >= K && (ldo & 7) == 0, "unfold_patches: ldo=%lld must be a multiple of 8 and >= C*p*p=%lld",
                 (long long)ldo, K);
  B200_CHECK_ARG(rows * ldo <= (1LL << 40) && (long long)B * oh <= 0x7fffffff && (long long)B * C * H * W <= (1LL << 40),
                 "unfold_patches: %lld patches too many", rows);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0 && (reinterpret_cast<uintptr_t>(img) & 1) == 0,
                 "unfold_patches: out_bf16 must be 16-byte aligned, img 2-byte aligned");
  B200_CHECK_ARG((size_t)p * p * sizeof(__nv_bfloat16) <= (size_t)kUnfoldSmem,
                 "unfold_patches: a %d x %d patch does not fit in shared memory", p, p);
  // all channels at once if one patch of them fits, else as many channels as fit; then as many patch columns as fit
  const long long per_c = (long long)p * sizeof(__nv_bfloat16);
  int cc = C;
  if (cc * per_c * p > kUnfoldSmem) cc = (int)(kUnfoldSmem / (per_c * p));
  const long long max_span = kUnfoldSmem / (per_c * cc);
  int nq = (int)((max_span - p) / s + 1);
  if (nq > ow) nq = ow;
  const size_t smem = (size_t)cc * p * ((nq - 1) * s + p) * sizeof(__nv_bfloat16);
  const dim3 grid((unsigned)(B * oh), (unsigned)((ow + nq - 1) / nq));
  B200_CHECK_ARG(grid.y <= 65535, "unfold_patches: %d patch columns too many", ow);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  unfold_kernel<<<grid, 256, smem, st>>>(reinterpret_cast<const __nv_bfloat16*>(img),
                                         reinterpret_cast<__nv_bfloat16*>(out_bf16), (long long)ldo, C, H, W, p, s, oh,
                                         ow, nq, cc);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_pit_pool(const float* x, int64_t M, int B, int h, int w, int D, const float* w9,
                                const float* bias, void* a_bf16, int64_t lda, void* cls_bf16, int64_t ldc,
                                void* stream) {
  B200_CHECK_ARG(x && w9 && bias && a_bf16 && cls_bf16, "pit_pool: null pointer");
  B200_CHECK_ARG(B > 0 && h > 0 && w > 0 && D > 0, "pit_pool: bad shape B=%d h=%d w=%d D=%d", B, h, w, D);
  B200_CHECK_ARG((long long)h * w <= (1LL << 24) && (long long)B * (h * w + 1) <= 0x7fffffff,
                 "pit_pool: %d x %d grid of %d images too large", h, w, B);
  B200_CHECK_ARG(M == (long long)B * (h * w + 1),
                 "pit_pool: x has %lld rows, B * (h*w + 1) = %lld expected (a cls row, then the h x w grid)",
                 (long long)M, (long long)B * (h * w + 1));
  B200_CHECK_ARG(D % 8 == 0, "pit_pool: D=%d must be a multiple of 8", D);
  B200_CHECK_ARG(lda >= 2 * D && (lda & 7) == 0 && ldc >= D && (ldc & 7) == 0,
                 "pit_pool: lda=%lld must be a multiple of 8 and >= 2D, ldc=%lld a multiple of 8 and >= D",
                 (long long)lda, (long long)ldc);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w9) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(bias) & 15) == 0 && (reinterpret_cast<uintptr_t>(a_bf16) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(cls_bf16) & 15) == 0,
                 "pit_pool: x, w9, bias, a_bf16 and cls_bf16 must be 16-byte aligned");
  int rb = 1;
  size_t smem = 0;
  const int ch = pool_tiling(h, w, D, &rb, &smem);
  B200_CHECK_ARG(ch > 0, "pit_pool: a grid row of %d tokens does not fit in shared memory", w);
  const int oh = (h + 1) / 2;
  const long long grid = (long long)B * ((oh + rb - 1) / rb);
  B200_CHECK_ARG(grid <= 0x7fffffff, "pit_pool: %lld CTAs too many", grid);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (ch) {
    case 32: launch_pool<32>((int)grid, smem, st, x, w9, bias, a_bf16, lda, cls_bf16, ldc, h, w, D, rb); break;
    case 16: launch_pool<16>((int)grid, smem, st, x, w9, bias, a_bf16, lda, cls_bf16, ldc, h, w, D, rb); break;
    default: launch_pool<8>((int)grid, smem, st, x, w9, bias, a_bf16, lda, cls_bf16, ldc, h, w, D, rb);
  }
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
