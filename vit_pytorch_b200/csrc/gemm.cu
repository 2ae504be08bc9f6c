// Persistent, warp-specialised bf16 GEMM for sm_90a:  out = epilogue(A[M,K] * W[N,K]^T)
//
//   warpgroup 0     : TMA producer  (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx)
//   warpgroups 1, 2 : consumers     (wgmma m64 x BLOCK_N x k16, fp32 accumulators in registers, 64 rows each), then
//                     the epilogue straight from the accumulator registers: bias / LN-fold / GELU / residual -> global
//
// The producer runs ahead into the next tile while the consumers finish the epilogue of the current one.
// Replaces the nn.Linear call sites listed in include/b200vit.h.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int NUM_THREADS = 384;

struct GemmParams {
  int M, N, K;
  int num_m_tiles, num_n_tiles, num_k_blocks;
  int flags;
  __nv_bfloat16* out_bf16;
  float* out_f32;
  long long ldo;
  const float* bias;
  const float* resid;
  const float* ln_sums;  // [M][ln_parts][2]
  int ln_parts;
  int stats_parts;
  int stats_width;       // output columns per statistics part (64 or 128)
  float ln_inv_dim;
  float ln_eps;
  const float* col_s;  // [N]
  float* stats_out;    // [M][stats_parts][2]
  // Rows of A (and of the output) per tile: BLOCK_M, or -- patch mode -- the patches of `patch_ght` patch rows of one
  // image (<= 128; the rest of the 128-row MMA tile is ignored).
  int rows_per_tile;
  // Patch mode (b200vit_patch_embed_tma): A is not a matrix in memory but the NCHW image itself, read through a 5-D
  // tensor map (pixel 16 | patch column | patch row | pixel row 16 | image x channel).  k block kb = channel * 4 + g
  // covers pixel rows 4g .. 4g+3 of every patch, loaded as four boxes of 16 pixels (32 bytes) per patch into four
  // 32B-swizzled slabs of 128 rows x 16 k: each slab is the K-major operand of one wgmma k-step.
  int patch;
  int patch_ght;            // patch rows per tile
  int patch_tiles_per_img;  // gh / patch_ght
  int patch_C;              // channels
};

// PATCH: the A stage holds FOUR 4 KB slabs, one per 16-wide k-step (see GemmParams::patch).
template <int BLOCK_N, int STAGES, bool PATCH = false>
struct GemmSmem {
  static constexpr int A_SLAB = PATCH ? BLOCK_M * 32 : BLOCK_M * BLOCK_K * 2;
  static constexpr int A_BYTES = PATCH ? 4 * A_SLAB : A_SLAB;
  static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  // full[STAGES], empty[STAGES]
  static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8;
  static constexpr int DYN_BYTES = TOTAL + 1024;  // slack for manual 1024B alignment
};

template <int BLOCK_N, int STAGES, bool PATCH>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p) {
  using L = GemmSmem<BLOCK_N, STAGES, PATCH>;
  constexpr int NACC = BLOCK_N / 2;          // fp32 accumulators per consumer thread (64 rows x BLOCK_N / 128)
  constexpr int CHUNKS = BLOCK_N / 64;       // 64-column statistics chunks per tile

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / p.num_n_tiles;
        const int n_blk = tile % p.num_n_tiles;
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          if (PATCH) {
            // im2col-free A tile: rows_per_tile patches x (4 pixel rows x 16 pixels) of channel kb / 4
            const int img = m_blk / p.patch_tiles_per_img, tin = m_blk % p.patch_tiles_per_img;
            mbar_arrive_expect_tx(&full_bar[stage], p.rows_per_tile * 128 + L::B_BYTES);
#pragma unroll
            for (int j = 0; j < 4; ++j)
              tma_load_5d(sa + j * L::A_SLAB, &tmA, &full_bar[stage], 0, 0, tin * p.patch_ght, (kb & 3) * 4 + j,
                          img * p.patch_C + (kb >> 2));
          } else {
            mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
            tma_load_2d(sa, &tmA, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
          }
          tma_load_2d(sb, &tmB, &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: MMA + epilogue
  setmaxnreg_inc<232>();
  const int c = wg - 1;                       // rows [64c, 64c + 64) of the tile
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const int flags = p.flags;
  const bool vec_ok = (p.ldo & 1) == 0;
  int stage = 0;
  uint32_t phase = 0;
  float acc[NACC];

  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m_blk = tile / p.num_n_tiles;
    const int n_blk = tile % p.num_n_tiles;

    int prev_stage = -1;
    for (int kb = 0; kb < p.num_k_blocks; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * L::STAGE_BYTES);
      const uint32_t sb = sa + L::A_BYTES;
      const uint64_t bdesc = make_wgmma_desc(sb, 1024, WGMMA_SW128);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
        // patch mode: the k-th 16 k of A are the 32-byte rows of slab k; otherwise +32 B inside the 128B swizzle row
        const uint64_t ad = PATCH ? make_wgmma_desc(sa + k * L::A_SLAB + c * 64 * 32, 256, WGMMA_SW32)
                                  : make_wgmma_desc(sa + c * 64 * 128, 1024, WGMMA_SW128) + 2 * k;
        if constexpr (BLOCK_N == 256) wgmma_m64n256k16(acc, ad, bdesc + 2 * k, (kb | k) != 0);
        else wgmma_m64n128k16(acc, ad, bdesc + 2 * k, (kb | k) != 0);
      }
      wgmma_commit();
      // the MMAs of the previous k block have finished reading their stage once at most one group is in flight
      wgmma_wait<1>();
      if (prev_stage >= 0 && t == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (t == 0) mbar_arrive(&empty_bar[prev_stage]);

    // ---------------------------------------------------------------- epilogue
    // accumulator layout (wgmma m64nN, fp32): acc[4j + h] holds row (16 warp + lane/4 + 8 (h >> 1)),
    // column (8 j + 2 (lane % 4) + (h & 1)) of this warpgroup's 64 x BLOCK_N block
    const int tr0 = c * 64 + warp * 16 + (lane >> 2);
    float mu[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f};
    int row[2];
    bool row_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int tr = tr0 + 8 * h;
      row[h] = m_blk * p.rows_per_tile + tr;
      row_ok[h] = row[h] < p.M && tr < p.rows_per_tile;
      if ((flags & B200VIT_EPI_LNFOLD) && row_ok[h]) {
        float s1 = 0.f, s2 = 0.f;
        for (int i = 0; i < p.ln_parts; ++i) {
          const float2 ss = *reinterpret_cast<const float2*>(p.ln_sums + 2 * ((size_t)row[h] * p.ln_parts + i));
          s1 += ss.x;
          s2 += ss.y;
        }
        mu[h] = s1 * p.ln_inv_dim;
        const float var = fmaxf(s2 * p.ln_inv_dim - mu[h] * mu[h], 0.f);
        rstd[h] = rsqrtf(var + p.ln_eps);
      }
    }
    float st_sum[2][CHUNKS], st_sq[2][CHUNKS];
#pragma unroll
    for (int q = 0; q < CHUNKS; ++q) st_sum[0][q] = st_sum[1][q] = st_sq[0][q] = st_sq[1][q] = 0.f;

    const int n0 = n_blk * BLOCK_N;
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int col = n0 + 8 * j + 2 * (lane & 3);
      if (col >= p.N) continue;
      const bool pair = vec_ok && col + 1 < p.N;
      float b0 = 0.f, b1 = 0.f, s0 = 0.f, s1 = 0.f;
      if (flags & B200VIT_EPI_BIAS) {
        b0 = p.bias[col];
        b1 = col + 1 < p.N ? p.bias[col + 1] : 0.f;
      }
      if (flags & B200VIT_EPI_LNFOLD) {
        s0 = p.col_s[col];
        s1 = col + 1 < p.N ? p.col_s[col + 1] : 0.f;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!row_ok[h]) continue;
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (flags & (B200VIT_EPI_LNFOLD | B200VIT_EPI_BIAS)) {
          // y = acc * rstd + (bias - rstd*mu * s)
          const bool fold = (flags & B200VIT_EPI_LNFOLD) != 0;
          const float k = -rstd[h] * mu[h];
          const float c0 = fold ? fmaf(k, s0, b0) : b0, c1 = fold ? fmaf(k, s1, b1) : b1;
          const float rs = fold ? rstd[h] : 1.0f;
          v0 = fmaf(v0, rs, c0);
          v1 = fmaf(v1, rs, c1);
        }
        if (flags & B200VIT_EPI_GELU) gelu_erf2(v0, v1);
        const size_t o = (size_t)row[h] * p.ldo + col;
        float r0 = 0.f, r1 = 0.f;
        if (pair) {
          if (flags & B200VIT_EPI_RESIDUAL) {
            const float2 rr = *reinterpret_cast<const float2*>(p.resid + o);
            v0 += rr.x;
            v1 += rr.y;
          }
          if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + o) = make_float2(v0, v1);
          const uint32_t pk = pack_bf16x2(v0, v1);
          if (p.out_bf16) *reinterpret_cast<uint32_t*>(p.out_bf16 + o) = pk;
          r0 = __uint_as_float(pk << 16);
          r1 = __uint_as_float(pk & 0xFFFF0000u);
        } else {
          // scalar tail (N or ldo odd)
          const float vv[2] = {v0, v1};
          float rr[2] = {0.f, 0.f};
          for (int i = 0; i < 2 && col + i < p.N; ++i) {
            float x = vv[i];
            if (flags & B200VIT_EPI_RESIDUAL) x += p.resid[o + i];
            if (p.out_f32) p.out_f32[o + i] = x;
            const __nv_bfloat16 xb = __float2bfloat16_rn(x);
            if (p.out_bf16) p.out_bf16[o + i] = xb;
            rr[i] = __bfloat162float(xb);
          }
          r0 = rr[0];
          r1 = rr[1];
        }
        if (flags & B200VIT_EPI_STATS) {
          st_sum[h][j / 8] += r0 + r1;
          st_sq[h][j / 8] = fmaf(r0, r0, fmaf(r1, r1, st_sq[h][j / 8]));
        }
      }
    }
    if (flags & B200VIT_EPI_STATS) {
      // the four lanes of a quad hold the same two rows: reduce, then lane 0 of the quad writes every part of the tile
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < CHUNKS; ++q) {
          st_sum[h][q] += __shfl_xor_sync(0xffffffffu, st_sum[h][q], 1);
          st_sum[h][q] += __shfl_xor_sync(0xffffffffu, st_sum[h][q], 2);
          st_sq[h][q] += __shfl_xor_sync(0xffffffffu, st_sq[h][q], 1);
          st_sq[h][q] += __shfl_xor_sync(0xffffffffu, st_sq[h][q], 2);
        }
      if ((lane & 3) == 0) {
        const int per = p.stats_width / 64;   // 64-column chunks per part
        const int first = n0 / p.stats_width;
        const int last = (n_blk == p.num_n_tiles - 1) ? p.stats_parts : first + CHUNKS / per;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!row_ok[h]) continue;
          float* so = p.stats_out + 2 * (size_t)row[h] * p.stats_parts;
          for (int part = first; part < last; ++part) {
            float a = 0.f, b = 0.f;
#pragma unroll
            for (int q = 0; q < CHUNKS; ++q)
              if (first + q / per == part) {
                a += st_sum[h][q];
                b += st_sq[h][q];
              }
            *reinterpret_cast<float2*>(so + 2 * part) = make_float2(a, b);
          }
        }
      }
    }
  }
}

// test hook 12: BLOCK_N of b200vit_gemm_bf16 -- 0 = auto (256 when N > 128), 1 = 128, 2 = 256
static std::atomic<int> g_gemm_block_n{0};
void gemm_set_block_n(int v) { g_gemm_block_n = v; }

template <int BLOCK_N, int STAGES, bool PATCH = false>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams& p, cudaStream_t stream) {
  using L = GemmSmem<BLOCK_N, STAGES, PATCH>;
  static_assert(L::DYN_BYTES <= 227 * 1024, "gemm: shared memory budget");
  auto kern = gemm_bf16_kernel<BLOCK_N, STAGES, PATCH>;
  B200_ENSURE_SMEM(kern, L::DYN_BYTES);
  if (!p.patch) p.rows_per_tile = BLOCK_M;
  p.num_m_tiles = (p.M + p.rows_per_tile - 1) / p.rows_per_tile;
  p.num_n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  p.num_k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
  p.stats_width = p.N > 128 ? 128 : 64;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, NUM_THREADS, L::DYN_BYTES, stream>>>(tmA, tmB, p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace b200

extern "C" int b200vit_stats_parts(int N) {
  const int block_n = N > 128 ? 256 : 128;      // two statistics parts per 256 (or, N <= 128, 128) columns
  return 2 * ((N + block_n - 1) / block_n);
}

extern "C" int b200vit_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* out_bf16,
                                 float* out_f32, int64_t ldo, const float* bias, const float* resid,
                                 const float* ln_sums, int ln_parts, float ln_eps, const float* col_s,
                                 float* stats_out, int M, int N, int K, int flags, void* stream) {
  using namespace b200;
  B200_CHECK_ARG(A && W, "gemm: A/W must not be null");
  B200_CHECK_ARG(out_bf16 || out_f32, "gemm: need at least one output");
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm: bad shape M=%d N=%d K=%d", M, N, K);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
                 "gemm: A and W must be 16-byte aligned");
  B200_CHECK_ARG((lda & 7) == 0 && (ldw & 7) == 0 && lda >= K && ldw >= K,
                 "gemm: lda=%lld ldw=%lld must be multiples of 8 and >= K=%d", (long long)lda, (long long)ldw, K);
  B200_CHECK_ARG(ldo >= N, "gemm: ldo=%lld < N=%d", (long long)ldo, N);
  B200_CHECK_ARG(!(flags & B200VIT_EPI_BIAS) || bias, "gemm: EPI_BIAS without bias");
  B200_CHECK_ARG(!(flags & B200VIT_EPI_RESIDUAL) || resid, "gemm: EPI_RESIDUAL without resid");
  B200_CHECK_ARG(!(flags & B200VIT_EPI_LNFOLD) || (ln_sums && col_s && ln_parts >= 1 && ln_parts <= 64),
                 "gemm: EPI_LNFOLD needs ln_sums, col_s and 1 <= ln_parts <= 64");
  B200_CHECK_ARG(!(flags & B200VIT_EPI_STATS) || stats_out, "gemm: EPI_STATS without stats_out");
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  B200_CHECK_ARG(al16(bias) && al16(resid) && al16(col_s) && al16(out_bf16) && al16(out_f32) && al16(ln_sums),
                 "gemm: epilogue pointers must be 16-byte aligned");

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);

  // K-tail: TMA zero-fills out-of-bounds columns of both operands, so any K works as long as rows are 16B multiples.
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.flags = flags;
  p.out_bf16 = reinterpret_cast<__nv_bfloat16*>(out_bf16);
  p.out_f32 = out_f32;
  p.ldo = ldo;
  p.bias = bias;
  p.resid = resid;
  p.ln_sums = ln_sums;
  p.ln_parts = ln_parts;
  p.stats_parts = b200vit_stats_parts(N);
  p.ln_inv_dim = 1.0f / (float)K;
  p.ln_eps = ln_eps;
  p.col_s = col_s;
  p.stats_out = stats_out;

  const int force = g_gemm_block_n.load();
  const bool wide = force == 0 ? N > 128 : force == 2;
  const uint32_t block_n = wide ? 256 : 128;
  CUtensorMap tmA, tmB;
  {
    const uint64_t dims[2] = {(uint64_t)K, (uint64_t)M};
    const uint64_t strides[1] = {(uint64_t)lda * 2};
    const uint32_t box[2] = {(uint32_t)BLOCK_K, (uint32_t)BLOCK_M};
    int rc = encode_tmap_bf16(&tmA, A, 2, dims, strides, box);
    if (rc) return rc;
  }
  {
    const uint64_t dims[2] = {(uint64_t)K, (uint64_t)N};
    const uint64_t strides[1] = {(uint64_t)ldw * 2};
    const uint32_t box[2] = {(uint32_t)BLOCK_K, block_n};
    int rc = encode_tmap_bf16(&tmB, W, 2, dims, strides, box);
    if (rc) return rc;
  }
  if (wide) return launch_gemm<256, 4>(tmA, tmB, p, st);
  return launch_gemm<128, 6>(tmA, tmB, p, st);
}

extern "C" int b200vit_rmsnorm_heads(void* buf, int64_t ld, const float* gamma, int T, int nheads, int dh, void* stream);
extern "C" int b200vit_layernorm_heads(void* buf, int64_t ld, const float* gamma, int T, int nheads, int dh, float eps,
                                       void* stream);

extern "C" int b200vit_gemm_headnorm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* out_bf16,
                                          int64_t ldo, const float* bias, const float* ln_sums, int ln_parts,
                                          float ln_eps, const float* col_s, const float* head_gamma, int norm_heads,
                                          int dh, float head_eps, int M, int N, int K, int flags, void* stream) {
  using namespace b200;
  B200_CHECK_ARG(out_bf16 && head_gamma, "gemm_headnorm: null pointer");
  B200_CHECK_ARG(dh == 64, "gemm_headnorm: dim_head=%d not supported by this build (only 64)", dh);
  B200_CHECK_ARG(norm_heads > 0 && norm_heads * 64 <= N, "gemm_headnorm: %d heads do not fit N=%d", norm_heads, N);
  B200_CHECK_ARG((flags & ~(B200VIT_EPI_BIAS | B200VIT_EPI_LNFOLD | B200VIT_EPI_HEADLN)) == 0,
                 "gemm_headnorm: unsupported flags %d", flags);
  const bool hln = (flags & B200VIT_EPI_HEADLN) != 0;
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(head_gamma) & 15) == 0, "gemm_headnorm: head_gamma must be 16-byte aligned");
  int rc = b200vit_gemm_bf16(A, lda, W, ldw, out_bf16, nullptr, ldo, bias, nullptr, ln_sums, ln_parts, ln_eps, col_s,
                             nullptr, M, N, K, flags & ~B200VIT_EPI_HEADLN, stream);
  if (rc) return rc;
  if (hln) return b200vit_layernorm_heads(out_bf16, ldo, head_gamma, M, norm_heads, dh, head_eps, stream);
  return b200vit_rmsnorm_heads(out_bf16, ldo, head_gamma, M, norm_heads, dh, stream);
}


// ------------------------------------------------------------------------------------------------------------------
// im2col-free patch embedding (p x p x C pixels staged through TMA into shared memory feed the wgmma GEMM directly):
// the patch projection reads the NCHW image directly; Rearrange('b c (h p1) (w p2) -> b (h w) (p1 p2 c)') and
// the LayerNorm over the patch (vit.py:100-101) never materialise.  LayerNorm is folded exactly like everywhere else:
//   LN(x) W^T + b  =  rstd (x (gamma W)^T - mu colsum) + (W beta + b),
// x = raw bf16 pixels (the A operand), (mu, rstd) from b200vit_patch_stats.  The K order of the operand is
// (c, p1, p2) -- the image's own order -- so the caller permutes the weight's columns from the reference's (p1 p2 c).
// ------------------------------------------------------------------------------------------------------------------
extern "C" int b200vit_patch_embed_tma(const void* img, const void* w_perm, const float* bias, const float* col_s,
                                       const float* patch_stats, float ln_eps, float* out_f32, int64_t ldo, int B, int C,
                                       int H, int W, int D, void* stream) {
  using namespace b200;
  B200_CHECK_ARG(img && w_perm && bias && col_s && patch_stats && out_f32, "patch_embed_tma: null pointer");
  B200_CHECK_ARG(B > 0 && C > 0 && C <= 8 && H > 0 && W > 0 && (H % 16) == 0 && (W % 16) == 0,
                 "patch_embed_tma: needs 16 x 16 patches on an image whose sides are multiples of 16 (got %dx%d)", H, W);
  B200_CHECK_ARG(D > 0 && (D % 8) == 0 && ldo >= D, "patch_embed_tma: bad D=%d / ldo", D);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(img) & 15) == 0 && (reinterpret_cast<uintptr_t>(w_perm) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(out_f32) & 15) == 0 && (reinterpret_cast<uintptr_t>(bias) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(col_s) & 15) == 0,
                 "patch_embed_tma: pointers must be 16-byte aligned");
  const int gh = H / 16, gw = W / 16;
  B200_CHECK_ARG(gw <= 128, "patch_embed_tma: %d patches per row do not fit a 128-row tile", gw);
  int ght = 1;  // largest divisor of gh whose patch rows fit the 128-row MMA tile
  for (int d = 1; d <= gh; ++d)
    if (gh % d == 0 && d * gw <= 128) ght = d;
  const int K = C * 256;
  GemmParams p{};
  p.M = B * gh * gw; p.N = D; p.K = K;
  p.flags = B200VIT_EPI_LNFOLD | B200VIT_EPI_BIAS;
  p.out_f32 = out_f32;
  p.ldo = ldo;
  p.bias = bias;
  p.ln_sums = patch_stats;
  p.ln_parts = 1;
  p.stats_parts = b200vit_stats_parts(D);
  p.ln_inv_dim = 1.0f / (float)K;
  p.ln_eps = ln_eps;
  p.col_s = col_s;
  p.patch = 1;
  p.patch_ght = ght;
  p.patch_tiles_per_img = gh / ght;
  p.patch_C = C;
  p.rows_per_tile = ght * gw;
  CUtensorMap tmA, tmB;
  {
    // innermost first: pixel in a patch row | patch column | patch row | pixel row in the patch | image x channel
    const uint64_t dims[5] = {16, (uint64_t)gw, (uint64_t)gh, 16, (uint64_t)B * C};
    const uint64_t strides[4] = {32, (uint64_t)16 * W * 2, (uint64_t)W * 2, (uint64_t)H * W * 2};
    const uint32_t box[5] = {16, (uint32_t)gw, (uint32_t)ght, 1, 1};
    int rc = encode_tmap_bf16_sw(&tmA, img, 5, dims, strides, box, 32);
    if (rc) return rc;
  }
  {
    const uint64_t dims[2] = {(uint64_t)K, (uint64_t)D};
    const uint64_t strides[1] = {(uint64_t)K * 2};
    const uint32_t box[2] = {(uint32_t)BLOCK_K, 256};
    int rc = encode_tmap_bf16(&tmB, w_perm, 2, dims, strides, box);
    if (rc) return rc;
  }
  return launch_gemm<256, 4, true>(tmA, tmB, p, reinterpret_cast<cudaStream_t>(stream));
}
