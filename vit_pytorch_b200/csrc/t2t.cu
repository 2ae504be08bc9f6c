// The operations of T2T-ViT (reference t2t.py) that no other kernel covers.
//
// b200vit_t2t_unfold_image / b200vit_t2t_unfold_tokens: one soft split, nn.Unfold(k, stride s, padding p) +
//   Rearrange('b c n -> b n c') (t2t.py:37-38), as bit copies into rows of out[B*oh*ow, ldo] (bf16: the A operand of
//   a GEMM; fp32: the residual stream of the soft-split Transformer that follows).  The source is the NCHW image
//   (first stage) or the bf16 token rows of the previous soft-split Transformer read as a map of int(sqrt(n)) rows
//   (RearrangeImage, t2t.py:20-22).  One CTA per output row; its threads walk the row in column order, so that every
//   warp writes one contiguous run (the output, up to round8(C*k*k) fp32 per row, is the larger side of the copy).  Columns [C*k*k, ldo) are zero filled.
//
// b200vit_attention_wide: softmax attention of one head as wide as the token (a soft-split Transformer, heads == 1 and
//   dim_head == dim, t2t.py:40) for heads too wide for a flash kernel's register-resident output (1344 fp32 columns of
//   128 rows would be 688 KB).  The scores are materialised per image instead, in three launches per chunk of images:
//     S = scale * Q K^T      batched wgmma GEMM over the packed qkv, fp32 scores in the workspace
//     P = softmax(S)         one warp per row, fp32, rounded to bf16 once
//     O = P V                batched wgmma GEMM, V read as the MN-major (transposed) B operand, as attention.cu does
//   The operands arrive by TMA through 3-D tensor maps (column, token, image), which zero-fill past each image's n
//   tokens, so no image reads another's rows.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

// ------------------------------------------------------------------------------------------------------------------
// soft-split unfold
// ------------------------------------------------------------------------------------------------------------------
// src(b, c, y, x) = src[b*sb + c*sc + y*sy + x*sx]; out row b*oh*ow + r*ow + q, column c*k*k + i*k + j =
// src(b, c, r*s - p + i, q*s - p + j), 0 where that falls outside the H x W map.
template <typename T>
__global__ void __launch_bounds__(256)
t2t_unfold_kernel(const __nv_bfloat16* __restrict__ src, long long sb, long long sc, long long sy, long long sx,
                  T* __restrict__ out, long long ldo, int C, int H, int W, int k, int s, int p, int oh, int ow) {
  const long long row = blockIdx.x;
  const int per_image = oh * ow;
  const int b = (int)(row / per_image), t = (int)(row - (long long)b * per_image);
  const int r = t / ow, q = t - r * ow;
  const int kk = k * k, K = C * kk;
  const __nv_bfloat16* img = src + (long long)b * sb;
  T* o = out + row * ldo;
  for (int e = threadIdx.x; e < K; e += blockDim.x) {
    const int c = e / kk, tap = e - c * kk;
    const int i = tap / k, j = tap - i * k;
    const int y = r * s - p + i, x = q * s - p + j;
    __nv_bfloat16 v = __float2bfloat16_rn(0.f);
    if (y >= 0 && y < H && x >= 0 && x < W) v = img[(long long)c * sc + (long long)y * sy + (long long)x * sx];
    if constexpr (sizeof(T) == 4) o[e] = __bfloat162float(v);
    else o[e] = v;
  }
  for (long long e = K + threadIdx.x; e < ldo; e += blockDim.x) {
    if constexpr (sizeof(T) == 4) o[e] = 0.f;
    else o[e] = __float2bfloat16_rn(0.f);
  }
}

static int launch_unfold(const void* src, long long sb, long long sc, long long sy, long long sx, void* out_bf16,
                         float* out_f32, int64_t ldo, int B, int C, int H, int W, int k, int s, int p,
                         cudaStream_t st) {
  const int oh = (H + 2 * p - k) / s + 1, ow = (W + 2 * p - k) / s + 1;
  const long long rows = (long long)B * oh * ow;
  const __nv_bfloat16* in = reinterpret_cast<const __nv_bfloat16*>(src);
  if (out_f32)
    t2t_unfold_kernel<float><<<(unsigned)rows, 256, 0, st>>>(in, sb, sc, sy, sx, out_f32, ldo, C, H, W, k, s, p, oh,
                                                             ow);
  else
    t2t_unfold_kernel<__nv_bfloat16><<<(unsigned)rows, 256, 0, st>>>(
        in, sb, sc, sy, sx, reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, C, H, W, k, s, p, oh, ow);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// wide attention: two batched wgmma GEMMs and a row softmax
// ------------------------------------------------------------------------------------------------------------------
// D[64 x 64] (+)= A * B, A K-major and B MN-major (transposed), both in shared memory
__device__ __forceinline__ void wgmma_m64n64k16_tb(float (&d)[32], uint64_t a_desc, uint64_t b_desc,
                                                   uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, 0, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

constexpr int WIDE_ROWS = 128;            // query rows of a CTA: two warpgroups of 64
constexpr int WIDE_THREADS = 256;
constexpr int WIDE_A_BYTES = WIDE_ROWS * 128;   // a 64-column slab of 128 rows (128B swizzle)
constexpr int WIDE_B_BYTES = 64 * 128;          // a 64-column slab of 64 rows
constexpr int WIDE_STAGE = WIDE_A_BYTES + WIDE_B_BYTES;
constexpr int WIDE_SMEM = 2 * WIDE_STAGE + 4 * 8 + 1024;

struct WideParams {
  int n, dp, z0;        // tokens per image, padded width, first image of the chunk in qkv
  int steps;            // 64-wide k steps: dp / 64 (scores) or key blocks (P V)
  float scale;
  float* S;             // scores [chunk][n][lds]
  long long lds;
  __nv_bfloat16* out;   // [B*n, dp] (may be null)
  float* x;             // residual stream (may be null), row pitch ldx, columns < n_resid
  long long ldx;
  int n_resid;
};

// One CTA = 128 query rows of image blockIdx.z of the chunk and one 64-wide output block (blockIdx.x): 64 keys of S
// (PV = false: A = the q slab, B = the k slab of k step c, both K-major) or 64 value columns of O (PV = true: A = the P
// tile of key block c, K-major, B = the v rows of that key block, MN-major).  Thread 0 loads both operands of every
// step with TMA into a two-stage ring, as attention.cu does; the 3-D maps (column, token, image) zero-fill past each
// image's n tokens.
template <bool PV>
__global__ void __launch_bounds__(WIDE_THREADS, 1)
t2t_wide_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const WideParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + 2 * WIDE_STAGE);
  uint64_t* empty = full + 2;
  const int z = blockIdx.z, q0 = blockIdx.y * WIDE_ROWS, c0 = blockIdx.x * 64;
  const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127, warp = t >> 5, lane = t & 31;

  auto issue = [&](int c) {
    const int st = c & 1;
    uint8_t* sb = smem + st * WIDE_STAGE;
    mbar_arrive_expect_tx(&full[st], WIDE_STAGE);
    if (PV) {
      tma_load_3d(sb, &tmA, &full[st], c * 64, q0, z);                              // P[z][q0 .., 64 c ..]
      tma_load_3d(sb + WIDE_A_BYTES, &tmB, &full[st], 2 * p.dp + c0, c * 64, p.z0 + z);   // v rows 64 c ..
    } else {
      tma_load_3d(sb, &tmA, &full[st], c * 64, q0, p.z0 + z);                       // q columns 64 c ..
      tma_load_3d(sb + WIDE_A_BYTES, &tmB, &full[st], p.dp + c * 64, c0, p.z0 + z);  // k rows c0 ..
    }
  };
  if (tid == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrive per warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    issue(0);
    if (p.steps > 1) issue(1);
  }
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  for (int c = 0; c < p.steps; ++c) {
    const int st = c & 1;
    const uint32_t ph = (c >> 1) & 1;
    mbar_wait(&full[st], ph);
    const uint32_t sa = smem_u32(smem + st * WIDE_STAGE) + wg * 64 * 128;
    const uint32_t sb = smem_u32(smem + st * WIDE_STAGE + WIDE_A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t ad = make_wgmma_desc(sa, 1024, WGMMA_SW128) + 2 * k;
      if (PV)
        wgmma_m64n64k16_tb(acc, ad, make_wgmma_desc_lbo(sb + k * 2048, 1024, 1024, WGMMA_SW128), 1);
      else
        wgmma_m64n64k16(acc, ad, make_wgmma_desc(sb, 1024, WGMMA_SW128) + 2 * k, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc);
    if (t == 0) mbar_arrive(&empty[st]);
    if (tid == 0 && c + 2 < p.steps) {
      mbar_wait(&empty[st], ph);  // both warpgroups are done with this stage
      issue(c + 2);
    }
  }

  // acc[4j + e]: row 16 warp + lane/4 + 8 (e >> 1) of the warpgroup's 64, column 8 j + 2 (lane % 4) + (e & 1)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = q0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * r;
    if (row >= p.n) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = c0 + 8 * j + 2 * (lane & 3);
      const float v0 = acc[4 * j + 2 * r], v1 = acc[4 * j + 2 * r + 1];
      if (!PV) {
        float* o = p.S + ((long long)z * p.n + row) * p.lds;
        if (col < p.n) o[col] = v0 * p.scale;
        if (col + 1 < p.n) o[col + 1] = v1 * p.scale;
      } else {
        const long long orow = (long long)(p.z0 + z) * p.n + row;
        const __nv_bfloat162 ob = __floats2bfloat162_rn(v0, v1);
        if (p.out) *reinterpret_cast<__nv_bfloat162*>(p.out + orow * p.dp + col) = ob;
        if (p.x) {
          float* x = p.x + orow * p.ldx;
          if (col < p.n_resid) x[col] += __low2float(ob);
          if (col + 1 < p.n_resid) x[col + 1] += __high2float(ob);
        }
      }
    }
  }
}

// P[z][i][0 .. ldp) = bf16(softmax(S[z][i][0 .. n))), zeros beyond n.  One warp per row; the row stays in registers.
constexpr int WIDE_SOFTMAX_PER_LANE = B200VIT_ATTN_WIDE_MAX_TOKENS / 32;
__global__ void __launch_bounds__(256)
t2t_wide_softmax_kernel(const float* __restrict__ S, long long lds, __nv_bfloat16* __restrict__ P, long long ldp,
                        long long rows, int n) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* s = S + row * lds;
  float v[WIDE_SOFTMAX_PER_LANE];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < WIDE_SOFTMAX_PER_LANE; ++i) {
    const int c = lane + 32 * i;
    v[i] = c < n ? s[c] : -INFINITY;
    mx = fmaxf(mx, v[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < WIDE_SOFTMAX_PER_LANE; ++i) {
    v[i] = lane + 32 * i < n ? expf(v[i] - mx) : 0.f;
    sum += v[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
  __nv_bfloat16* pr = P + row * ldp;
#pragma unroll
  for (int i = 0; i < WIDE_SOFTMAX_PER_LANE; ++i) {
    const int c = lane + 32 * i;
    if (c < ldp) pr[c] = __float2bfloat16_rn(v[i] * inv);
  }
}

static long long round_up(long long a, long long b) { return (a + b - 1) / b * b; }

}  // namespace b200

using namespace b200;

extern "C" int b200vit_t2t_unfold_image(const void* img, void* out_bf16, float* out_f32, int64_t ldo, int B, int C,
                                        int H, int W, int k, int s, int p, void* stream) {
  B200_CHECK_ARG(img && (out_bf16 != nullptr) != (out_f32 != nullptr),
                 "t2t_unfold_image: null image, or not exactly one of out_bf16 / out_f32");
  B200_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && k >= 1 && s >= 1 && p >= 0 && p < k,
                 "t2t_unfold_image: bad shape B=%d C=%d H=%d W=%d k=%d s=%d p=%d", B, C, H, W, k, s, p);
  B200_CHECK_ARG(H + 2 * p >= k && W + 2 * p >= k, "t2t_unfold_image: %d x %d image smaller than one %d x %d window", H,
                 W, k, k);
  const long long K = (long long)C * k * k;
  B200_CHECK_ARG(ldo >= K && (ldo & 7) == 0, "t2t_unfold_image: ldo=%lld must be a multiple of 8 and >= C*k*k=%lld",
                 (long long)ldo, K);
  const long long rows = (long long)B * ((H + 2 * p - k) / s + 1) * ((W + 2 * p - k) / s + 1);
  B200_CHECK_ARG(rows <= 0x7fffffffLL, "t2t_unfold_image: %lld output rows too many", rows);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(img) & 1) == 0 && (reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(out_f32) & 15) == 0,
                 "t2t_unfold_image: out must be 16-byte aligned");
  return launch_unfold(img, (long long)C * H * W, (long long)H * W, W, 1, out_bf16, out_f32, ldo, B, C, H, W, k, s, p,
                       reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b200vit_t2t_unfold_tokens(const void* x, int64_t ldx, int B, int n, int C, void* out_bf16,
                                         float* out_f32, int64_t ldo, int k, int s, int p, void* stream) {
  B200_CHECK_ARG(x && (out_bf16 != nullptr) != (out_f32 != nullptr),
                 "t2t_unfold_tokens: null input, or not exactly one of out_bf16 / out_f32");
  B200_CHECK_ARG(B > 0 && n > 0 && C > 0 && k >= 1 && s >= 1 && p >= 0 && p < k,
                 "t2t_unfold_tokens: bad shape B=%d n=%d C=%d k=%d s=%d p=%d", B, n, C, k, s, p);
  B200_CHECK_ARG(ldx >= C, "t2t_unfold_tokens: ldx=%lld < C=%d", (long long)ldx, C);
  int h = 0;
  while ((long long)(h + 1) * (h + 1) <= n) ++h;  // int(sqrt(n)), t2t.py:22
  B200_CHECK_ARG(n % h == 0, "t2t_unfold_tokens: %d tokens cannot be read as a map of %d rows (t2t.py:22)", n, h);
  const int w = n / h;
  B200_CHECK_ARG(h + 2 * p >= k && w + 2 * p >= k, "t2t_unfold_tokens: %d x %d map smaller than one %d x %d window", h,
                 w, k, k);
  const long long K = (long long)C * k * k;
  B200_CHECK_ARG(ldo >= K && (ldo & 7) == 0, "t2t_unfold_tokens: ldo=%lld must be a multiple of 8 and >= C*k*k=%lld",
                 (long long)ldo, K);
  const long long rows = (long long)B * ((h + 2 * p - k) / s + 1) * ((w + 2 * p - k) / s + 1);
  B200_CHECK_ARG(rows <= 0x7fffffffLL, "t2t_unfold_tokens: %lld output rows too many", rows);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 1) == 0 && (reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(out_f32) & 15) == 0,
                 "t2t_unfold_tokens: out must be 16-byte aligned");
  return launch_unfold(x, (long long)n * ldx, 1, (long long)w * ldx, ldx, out_bf16, out_f32, ldo, B, C, h, w, k, s, p,
                       reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int64_t b200vit_attention_wide_workspace(int n, int dp, int images) {
  if (n <= 0 || images <= 0) return 0;
  (void)dp;
  const long long per_image = (long long)n * round_up(n, 4) * 4 + (long long)n * round_up(n, 64) * 2;
  return per_image * images + 2048;   // the workspace's and P's 1024-byte alignment
}

extern "C" int b200vit_attention_wide(const void* qkv, void* out, float* x, int64_t ldx, int n_resid, int B, int n,
                                      int dp, float scale, void* ws, int64_t ws_bytes, void* stream) {
  B200_CHECK_ARG(qkv && ws && (out || x), "attention_wide: null pointer (qkv, ws, and out or x)");
  B200_CHECK_ARG(B > 0 && n > 0 && n <= B200VIT_ATTN_WIDE_MAX_TOKENS,
                 "attention_wide: B=%d, n=%d tokens per image (1 .. %d)", B, n, B200VIT_ATTN_WIDE_MAX_TOKENS);
  B200_CHECK_ARG(dp > 0 && dp % 64 == 0 && dp <= B200VIT_ATTN_WIDE_MAX_WIDTH,
                 "attention_wide: head width dp=%d must be a multiple of 64 and <= %d", dp,
                 B200VIT_ATTN_WIDE_MAX_WIDTH);
  B200_CHECK_ARG(!x || (n_resid > 0 && n_resid <= dp && ldx >= n_resid),
                 "attention_wide: residual columns n_resid=%d must be in 1 .. dp=%d and <= ldx=%lld", n_resid, dp,
                 (long long)ldx);
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  B200_CHECK_ARG(al16(qkv) && al16(out) && al16(ws) && (reinterpret_cast<uintptr_t>(x) & 3) == 0,
                 "attention_wide: qkv, out and ws must be 16-byte aligned");
  const long long lds = round_up(n, 4), ldp = round_up(n, 64);
  const long long per_image = (long long)n * lds * 4 + (long long)n * ldp * 2;
  long long chunk = (ws_bytes - 2048) / per_image;
  B200_CHECK_ARG(chunk >= 1, "attention_wide: a workspace of %lld bytes holds no image (%lld needed per image)",
                 (long long)ws_bytes, per_image + 2048);
  if (chunk > B) chunk = B;
  if (chunk > 65535) chunk = 65535;
  B200_CHECK_ARG((long long)B * n * 3 * dp <= (1LL << 40), "attention_wide: qkv too large");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 1023) & ~uintptr_t(1023));
  float* S = reinterpret_cast<float*>(base);
  __nv_bfloat16* P = reinterpret_cast<__nv_bfloat16*>(base + round_up(chunk * n * lds * 4, 1024));
  // qkv as (column, token, image): q / k / v slabs of 128 or 64 token rows; P as (key, query, image of the chunk)
  CUtensorMap tmQ, tmKV, tmP;
  {
    const uint64_t dims[3] = {(uint64_t)3 * dp, (uint64_t)n, (uint64_t)B};
    const uint64_t strides[2] = {(uint64_t)3 * dp * 2, (uint64_t)3 * dp * 2 * n};
    const uint32_t qbox[3] = {64, WIDE_ROWS, 1}, kvbox[3] = {64, 64, 1};
    int rc = encode_tmap_bf16(&tmQ, qkv, 3, dims, strides, qbox);
    if (!rc) rc = encode_tmap_bf16(&tmKV, qkv, 3, dims, strides, kvbox);
    if (rc) return rc;
  }
  {
    const uint64_t dims[3] = {(uint64_t)ldp, (uint64_t)n, (uint64_t)chunk};
    const uint64_t strides[2] = {(uint64_t)ldp * 2, (uint64_t)ldp * 2 * n};
    const uint32_t box[3] = {64, WIDE_ROWS, 1};
    int rc = encode_tmap_bf16(&tmP, P, 3, dims, strides, box);
    if (rc) return rc;
  }
  B200_ENSURE_SMEM(t2t_wide_gemm_kernel<false>, WIDE_SMEM);
  B200_ENSURE_SMEM(t2t_wide_gemm_kernel<true>, WIDE_SMEM);
  const int qtiles = (n + WIDE_ROWS - 1) / WIDE_ROWS;
  for (long long z0 = 0; z0 < B; z0 += chunk) {
    const int nz = (int)(B - z0 < chunk ? B - z0 : chunk);
    WideParams p{};
    p.n = n;
    p.dp = dp;
    p.z0 = (int)z0;
    p.scale = scale;
    p.S = S;
    p.lds = lds;
    p.steps = dp / 64;
    t2t_wide_gemm_kernel<false><<<dim3((n + 63) / 64, qtiles, nz), WIDE_THREADS, WIDE_SMEM, st>>>(tmQ, tmKV, p);
    B200_CHECK_CUDA(cudaGetLastError());
    const long long srows = (long long)nz * n;
    t2t_wide_softmax_kernel<<<(unsigned)((srows + 7) / 8), 256, 0, st>>>(S, lds, P, ldp, srows, n);
    B200_CHECK_CUDA(cudaGetLastError());
    p.steps = (n + 63) / 64;
    p.out = reinterpret_cast<__nv_bfloat16*>(out);
    p.x = x;
    p.ldx = ldx;
    p.n_resid = n_resid;
    t2t_wide_gemm_kernel<true><<<dim3(dp / 64, qtiles, nz), WIDE_THREADS, WIDE_SMEM, st>>>(tmP, tmKV, p);
    B200_CHECK_CUDA(cudaGetLastError());
    count_launch(3);
  }
  return 0;
}
