// Persistent, warp-specialised bf16 GEMM for sm_90a:  out = epilogue(A[M,K] * W[N,K]^T)
//
//   warpgroup 0     : loaders
//                     warp 0 (one thread): A / W tiles, cp.async.bulk.tensor -> 128B-swizzled smem ring
//                     warp 1 (one thread, residual GEMMs only): the fp32 residual tile, TMA -> two 64-column slab
//                     buffers (256-wide tiles with TMA stores: none; warp 0 loads the four slabs into the four ring
//                     stages after the tile's last k block)
//                     warp 2: the tile's bias / col_s slices and LN-fold row sums -> smem (double buffered per tile)
//   warpgroups 1, 2 : consumers     (wgmma m64 x BLOCK_N x k16, fp32 accumulators in registers, 64 rows each), then
//                     the epilogue from the accumulator registers: bias / LN-fold / GELU / residual
//
// The loaders run ahead into the next tile while the consumers finish the epilogue of the current one, so every
// epilogue input is already in shared memory when the accumulators are ready.  (Read from global memory inside the
// epilogue, each residual load would wait behind the previous column's stores -- resid may be out_f32 itself -- for a
// full memory latency.)
// The outputs leave through shared memory too, written by TMA stores that drain while the consumers go on.  Written
// from the registers instead, every warp store puts 16 bytes into each of 8 rows, and the tile is bound by the rate of
// store instructions, not by HBM.
//   bf16 output (QKV, FC1): the epilogue writes 128B-swizzled staging boxes of 64 x 64 for the whole tile, one thread
//     per warpgroup hands them to TMA stores, and the consumers go straight on to the next tile's MMAs.  Thread 0 waits
//     for the stores to have read the staging tile during the next tile's first k block, before it is written again.
//   residual (out-proj, FC2): the fp32 sum goes back into the residual slab at the address its residual was read
//     from and is TMA-stored from there; once the previous slab's stores have read the one 16 KB staging chunk, the
//     bf16 copy is rounded from those sums into it.  A slab returns to its loader once its stores have read it: at the
//     next slab, or during the next tile's first k block.  Out-proj and FC2 run 256-wide tiles when the grid has at
//     least one per SM; their vector buffer holds the bias slice alone, so residual launches with an LN fold stay
//     128 wide.
// The direct-store epilogue remains for non-residual fp32 outputs, patch tiles of fewer than 128 rows, ldo or N not a
// multiple of 8, 256-wide residual tiles with an LN fold (test hook 12) and every launch under test hook 14.
// Replaces the nn.Linear call sites listed in include/b200vit.h.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int NUM_THREADS = 384;
constexpr int NUM_CONSUMERS = 256;

struct GemmParams {
  int M, N, K;
  int num_m_tiles, num_n_tiles, num_k_blocks;
  int flags;
  __nv_bfloat16* out_bf16;
  float* out_f32;
  long long ldo;
  const float* bias;
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
// RES (EPI_RESIDUAL launches): two residual slabs of 128 rows x 64 fp32 columns after the ring.  A slab is two TMA
// boxes of 32 columns (128 B per row, 128B swizzle: 16-byte chunk c of row r sits at chunk c ^ (r % 8)), so that the
// epilogue's float2 reads -- 8 rows x 4 column pairs per warp instruction -- touch every bank exactly twice.
// TMA_OUT: the bf16 output is staged in 128B-swizzled boxes of 64 rows x 64 columns (8 KB) and written by TMA stores.
// Without RES that is the whole tile (consumer warpgroup c owns boxes [c * BLOCK_N / 64, (c + 1) * BLOCK_N / 64)); with
// RES one 128 x 64 chunk, the bf16 copy of the slab being stored (warpgroup c owns its c-th box), while the fp32 sums
// go back into the residual slab they were read from and are stored from there.
// BIAS_ONLY (256-wide residual tiles with TMA stores): the vector buffer holds the bias slice alone, once; such
// launches never carry an LN fold.
template <int BLOCK_N, int STAGES, bool PATCH = false, bool RES = false, bool TMA_OUT = false>
struct GemmSmem {
  static constexpr bool BIAS_ONLY = RES && TMA_OUT && BLOCK_N == 256;
  // ... and its four slabs load into the ring, a 32 KB slab per 48 KB stage, under the tile's last k blocks: with no
  // slab buffers the ring has 4 stages instead of 3
  static constexpr bool RING_SLABS = BIAS_ONLY;
  static constexpr int BUF_SLABS = RING_SLABS ? 0 : BLOCK_N / 64;  // slabs of a tile in the two slab buffers
  static constexpr int A_SLAB = PATCH ? BLOCK_M * 32 : BLOCK_M * BLOCK_K * 2;
  static constexpr int A_BYTES = PATCH ? 4 * A_SLAB : A_SLAB;
  static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RES_BOX = BLOCK_M * 32 * 4;
  static constexpr int RES_SLAB = 2 * RES_BOX;
  static constexpr int RES_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int OUT_BOX = 64 * 64 * 2;
  static constexpr int OUT_OFFSET = RES_OFFSET + (RES && !RING_SLABS ? 2 * RES_SLAB : 0);
  static constexpr int OUT_BYTES = !TMA_OUT ? 0 : RES ? 2 * OUT_BOX : BLOCK_M * BLOCK_N * 2;
  // per tile, double buffered: bias[BLOCK_N], col_s[BLOCK_N], LN-fold row sums [BLOCK_M][2] (BIAS_ONLY: bias[BLOCK_N],
  // one buffer)
  static constexpr int VEC_OFFSET = OUT_OFFSET + OUT_BYTES;
  static constexpr int VEC_BYTES = (BIAS_ONLY ? BLOCK_N : 2 * BLOCK_N + 2 * BLOCK_M) * 4;
  static constexpr int VEC_BUFS = BIAS_ONLY ? 1 : 2;
  static constexpr int BAR_OFFSET = VEC_OFFSET + VEC_BUFS * VEC_BYTES;
  // full[STAGES], empty[STAGES], res_full[2], res_empty[2], vec_full[2], vec_empty[2]
  static constexpr int TOTAL = BAR_OFFSET + (2 * STAGES + 8) * 8;
  static constexpr int DYN_BYTES = TOTAL + 1024;  // slack for manual 1024B alignment
};

// named barrier over the 128 threads of one consumer warpgroup (ids 1, 2; 0 is __syncthreads)
// (the id comes from a register, so ptxas reserves all 16 named barriers; harmless at one CTA per SM)
__device__ __forceinline__ void warpgroup_sync(int c) { asm volatile("bar.sync %0, 128;" ::"r"(c + 1) : "memory"); }

// tmO / tmF (TMA_OUT only): store maps over out_bf16 (64 x 64 boxes) and out_f32 (32 x 64 boxes), 128B swizzle
// SIG: the instances that take EPI_SILU / EPI_SIGMOID (the squeeze-excitation GEMMs); every other instance is compiled
// without that branch
// EPI >= 0 (TMA_OUT only): the instance runs launches whose flags are exactly EPI -- the encoder layer's flag sets, see
// launch_tma_out -- so that every flag test of the epilogue is resolved at compile time; -1: the flags of the launch
template <int BLOCK_N, int STAGES, bool PATCH, bool RES, bool TMA_OUT, bool SIG = false, int EPI = -1>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmO,
                 const __grid_constant__ CUtensorMap tmF, const GemmParams p) {
  static_assert(!(TMA_OUT && PATCH), "patch tiles have fewer than 128 rows: a 64-row box would overwrite the next one");
  static_assert(EPI < 0 || (TMA_OUT && !SIG), "compiled flag sets are for the TMA-store epilogue");
  using L = GemmSmem<BLOCK_N, STAGES, PATCH, RES, TMA_OUT>;
  constexpr int NACC = BLOCK_N / 2;          // fp32 accumulators per consumer thread (64 rows x BLOCK_N / 128)
  constexpr int CHUNKS = BLOCK_N / 64;       // 64-column statistics chunks (and residual slabs) per tile

  extern __shared__ uint8_t smem_raw[];
  // offset from the __shared__ array itself (no round trip through an integer), so that the compiler knows every
  // access below is to shared memory and may schedule the epilogue's smem reads ahead of its global stores
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* res_full = empty_bar + STAGES;
  uint64_t* res_empty = res_full + 2;
  uint64_t* vec_full = res_empty + 2;
  uint64_t* vec_empty = vec_full + 2;

  const int wg = threadIdx.x >> 7;
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (RES) tma_prefetch_desc(&tmR);
    if (TMA_OUT && p.out_bf16) tma_prefetch_desc(&tmO);
    if (TMA_OUT && RES && p.out_f32) tma_prefetch_desc(&tmF);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(&res_full[s], 1);
      // TMA_OUT: thread 0 of each consumer warpgroup, once the stores of its half of the slab have read it
      mbar_init(&res_empty[s], TMA_OUT ? 2 : NUM_CONSUMERS);
      mbar_init(&vec_full[s], 64);  // every thread of loader warps 2 and 3
      mbar_init(&vec_empty[s], NUM_CONSUMERS);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ loaders
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
        if (L::RING_SLABS) {
          const int n0 = n_blk * BLOCK_N;
          const int nslab = min(BLOCK_N / 64, (p.N - n0 + 63) / 64);
          for (int q = L::BUF_SLABS; q < nslab; ++q) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            const int c0 = n0 + 64 * q;
            const int nbox = c0 + 32 < p.N ? 2 : 1;
            mbar_arrive_expect_tx(&full_bar[stage], nbox * L::RES_BOX);
            uint8_t* slab = smem + stage * L::STAGE_BYTES;
            for (int b = 0; b < nbox; ++b)
              tma_load_2d(slab + b * L::RES_BOX, &tmR, &full_bar[stage], c0 + 32 * b, m_blk * BLOCK_M);
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    } else if (RES && threadIdx.x == 32) {
      // residual slabs: the consumers release slab q of a tile after its last column group, so the first two slabs
      // of a tile load during the tile's main loop.  Boxes wholly right of N are not loaded (nor waited for).
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n0 = (tile % p.num_n_tiles) * BLOCK_N;
        const int m0 = (tile / p.num_n_tiles) * BLOCK_M;
        const int nslab = min(L::BUF_SLABS, (p.N - n0 + 63) / 64);
        for (int q = 0; q < nslab; ++q, ++it) {
          const int buf = it & 1;
          mbar_wait(&res_empty[buf], ((it >> 1) & 1) ^ 1);
          const int c0 = n0 + 64 * q;
          const int nbox = c0 + 32 < p.N ? 2 : 1;
          mbar_arrive_expect_tx(&res_full[buf], nbox * L::RES_BOX);
          uint8_t* slab = smem + L::RES_OFFSET + buf * L::RES_SLAB;
          for (int b = 0; b < nbox; ++b) tma_load_2d(slab + b * L::RES_BOX, &tmR, &res_full[buf], c0 + 32 * b, m0);
        }
      }
    } else if ((threadIdx.x >> 5) >= 2) {
      // warp 2: the tile's bias / col_s slices (zero past N); warp 3: its rows' LN-fold sums (added up in part order)
      const int lane = threadIdx.x & 31;
      const bool vec_warp = (threadIdx.x >> 5) == 2;
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        const int m_blk = tile / p.num_n_tiles;
        const int n0 = (tile % p.num_n_tiles) * BLOCK_N;
        const int vb = it % L::VEC_BUFS;
        mbar_wait(&vec_empty[vb], ((it / L::VEC_BUFS) & 1) ^ 1);
        float* vbias = reinterpret_cast<float*>(smem + L::VEC_OFFSET + vb * L::VEC_BYTES);
        float* vcs = vbias + BLOCK_N;
        float2* vln = reinterpret_cast<float2*>(vcs + BLOCK_N);
        if (vec_warp) {
#pragma unroll
          for (int i = lane; i < BLOCK_N; i += 32) {
            const int col = n0 + i;
            vbias[i] = (p.flags & B200VIT_EPI_BIAS) && col < p.N ? p.bias[col] : 0.f;
            if (!L::BIAS_ONLY) vcs[i] = (p.flags & B200VIT_EPI_LNFOLD) && col < p.N ? p.col_s[col] : 0.f;
          }
        } else if (!L::BIAS_ONLY && (p.flags & B200VIT_EPI_LNFOLD)) {
          float s1[BLOCK_M / 32], s2[BLOCK_M / 32];
          bool ok[BLOCK_M / 32];
#pragma unroll
          for (int k = 0; k < BLOCK_M / 32; ++k) {
            const int tr = lane + 32 * k;
            ok[k] = m_blk * p.rows_per_tile + tr < p.M && tr < p.rows_per_tile;
            s1[k] = s2[k] = 0.f;
          }
#pragma unroll 1  // four loads in flight per lane fit the loaders' 40 registers
          for (int i = 0; i < p.ln_parts; ++i)
#pragma unroll
            for (int k = 0; k < BLOCK_M / 32; ++k)
              if (ok[k]) {
                const size_t row = (size_t)m_blk * p.rows_per_tile + lane + 32 * k;
                const float2 ss = *reinterpret_cast<const float2*>(p.ln_sums + 2 * (row * p.ln_parts + i));
                s1[k] += ss.x;
                s2[k] += ss.y;
              }
#pragma unroll
          for (int k = 0; k < BLOCK_M / 32; ++k) vln[lane + 32 * k] = make_float2(s1[k], s2[k]);
        }
        mbar_arrive(&vec_full[vb]);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: MMA + epilogue
  setmaxnreg_inc<232>();
  const int c = wg - 1;                       // rows [64c, 64c + 64) of the tile
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  // (BIAS_ONLY: the host routes LN folds elsewhere)
  const int flags = EPI >= 0 ? EPI : L::BIAS_ONLY ? p.flags & ~B200VIT_EPI_LNFOLD : p.flags;
  const bool vec_ok = (p.ldo & 1) == 0;
  int stage = 0;
  uint32_t phase = 0;
  int slab_it = 0;  // residual slabs consumed so far (the loader's count)
  // TMA_OUT && RES, thread 0: the slab its stores may still be reading, as the index of its empty barrier from
  // empty_bar (a ring stage s: s; slab buffer b: STAGES + 2 + b, past res_full), or -1
  int pend_slab = -1;
  uint8_t* const stg_wg = smem + L::OUT_OFFSET + c * (RES ? L::OUT_BOX : 64 * BLOCK_N * 2);
  float acc[NACC];

  for (int tile = blockIdx.x, it = 0; tile < num_tiles; tile += gridDim.x, ++it) {
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
      // while the first MMAs run: the previous tile's output stores have read the staging tile (RES: and the last
      // slab, which goes back to the residual loader so that it can fill it during this main loop)
      if (TMA_OUT && kb == 0 && t == 0) {
        tma_store_wait_read<0>();
        if (RES && pend_slab >= 0) mbar_arrive(&empty_bar[pend_slab]);
        pend_slab = -1;
      }
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
    if (TMA_OUT && !RES) warpgroup_sync(c);  // ... and the whole warpgroup may write it again

    // ---------------------------------------------------------------- epilogue
    // accumulator layout (wgmma m64nN, fp32): acc[4j + h] holds row (16 warp + lane/4 + 8 (h >> 1)),
    // column (8 j + 2 (lane % 4) + (h & 1)) of this warpgroup's 64 x BLOCK_N block
    const int tr0 = c * 64 + warp * 16 + (lane >> 2);
    const int vb = it % L::VEC_BUFS;
    mbar_wait(&vec_full[vb], (it / L::VEC_BUFS) & 1);
    const float* vbias = reinterpret_cast<const float*>(smem + L::VEC_OFFSET + vb * L::VEC_BYTES);
    const float* vcs = vbias + BLOCK_N;
    const float2* vln = reinterpret_cast<const float2*>(vcs + BLOCK_N);
    float mu[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f};
    int row[2];
    bool row_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int tr = tr0 + 8 * h;
      row[h] = m_blk * p.rows_per_tile + tr;
      row_ok[h] = row[h] < p.M && tr < p.rows_per_tile;
      if ((flags & B200VIT_EPI_LNFOLD) && row_ok[h]) {
        const float2 ss = vln[tr];
        const float s1 = ss.x, s2 = ss.y;
        mu[h] = s1 * p.ln_inv_dim;
        const float var = fmaxf(s2 * p.ln_inv_dim - mu[h] * mu[h], 0.f);
        rstd[h] = rsqrtf(var + p.ln_eps);
      }
    }
    float st_sum[2][CHUNKS], st_sq[2][CHUNKS];
#pragma unroll
    for (int q = 0; q < CHUNKS; ++q) st_sum[0][q] = st_sum[1][q] = st_sq[0][q] = st_sq[1][q] = 0.f;

    const int n0 = n_blk * BLOCK_N;
    const int nslab = RES ? min(CHUNKS, (p.N - n0 + 63) / 64) : 0;
    // this thread's float2 in a residual slab: row tr0 (+ 8 h), 16-byte chunk (2 (j % 4) + (lane & 3) / 2) ^ (tr0 % 8)
    // of box (j % 8) / 4, 8-byte half lane & 1
    const int res_off = tr0 * 128 + (lane & 1) * 8;
    const int res_xor = ((lane & 3) >> 1) ^ (lane >> 2);
    // TMA_OUT: this thread's bf16 pair in a staging box: row tr0 % 64 (+ 8 h), 16-byte chunk (j % 8) ^ (tr0 % 8),
    // byte 4 (lane % 4) -- the 8 rows of a warp store land in 8 different chunks, so the stores are conflict free
    const int stg_off = (tr0 - 64 * c) * 128 + 4 * (lane & 3);
    // GUARD: skip the pairs outside M x N.  A compiled flag set without a residual needs no such test: whatever lands
    // in the staging tile past M or N stays there, because the store maps clip both edges, and these flag sets collect
    // no statistics.  (It is finite, too: TMA zero-fills A and W outside their maps, vbias / vcs are zero past N, and
    // the LN sums of rows past M are zero, so their rstd is rsqrt(eps).)  With a residual, a slab's columns past N
    // hold stale data that would enter the row statistics.  Without the tests, and with the flags known at compile
    // time, the loop is straight-line code whose pairs the compiler interleaves.
    constexpr bool GUARD = EPI < 0 || RES;
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int pc = 8 * j + 2 * (lane & 3);  // column of the pair in the tile
      const int col = n0 + pc;
      // RING_SLABS: the slabs sit in the ring stages after the tile's last k block
      const bool ring_slab = L::RING_SLABS && j / 8 >= L::BUF_SLABS;
      if (RES && j % 8 == 0 && j / 8 < nslab) {
        if (ring_slab) mbar_wait(&full_bar[stage], phase);
        else mbar_wait(&res_full[slab_it & 1], (slab_it >> 1) & 1);
      }
      uint8_t* const slab_base =
          smem + (ring_slab ? stage * L::STAGE_BYTES : L::RES_OFFSET + (slab_it & 1) * L::RES_SLAB);
      uint8_t* slab = slab_base + ((j % 8) / 4) * L::RES_BOX + res_off;
      uint8_t* stg = stg_wg + (RES ? 0 : (j / 8) * L::OUT_BOX) + stg_off + (((j % 8) ^ (lane >> 2)) << 4);
      const bool pair = vec_ok && col + 1 < p.N;
      float b0 = 0.f, b1 = 0.f, s0 = 0.f, s1 = 0.f;
      if (flags & B200VIT_EPI_BIAS) {
        const float2 bb = *reinterpret_cast<const float2*>(vbias + pc);
        b0 = bb.x;
        b1 = bb.y;
      }
      if (flags & B200VIT_EPI_LNFOLD) {
        const float2 ss = *reinterpret_cast<const float2*>(vcs + pc);
        s0 = ss.x;
        s1 = ss.y;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (GUARD && (!row_ok[h] || col >= p.N)) continue;
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
        if (flags & B200VIT_EPI_HARDSWISH) {  // y * clamp(y + 3, 0, 6) / 6 (nn.Hardswish, levit.py:32)
          v0 = v0 * fminf(fmaxf(v0 + 3.0f, 0.0f), 6.0f) * (1.0f / 6.0f);
          v1 = v1 * fminf(fmaxf(v1 + 3.0f, 0.0f), 6.0f) * (1.0f / 6.0f);
        }
        if (SIG && (flags & (B200VIT_EPI_SILU | B200VIT_EPI_SIGMOID))) {
          // sigmoid(y) = 1 / (1 + 2^(-y log2 e)) (nn.Sigmoid, max_vit.py:57); SiLU is y sigmoid(y) (max_vit.py:55)
          const float g0 = fast_rcp(1.0f + fast_ex2(-1.4426950408889634f * v0));
          const float g1 = fast_rcp(1.0f + fast_ex2(-1.4426950408889634f * v1));
          const bool silu = (flags & B200VIT_EPI_SILU) != 0;
          v0 = silu ? v0 * g0 : g0;
          v1 = silu ? v1 * g1 : g1;
        }
        const size_t o = (size_t)row[h] * p.ldo + col;
        float2* rp = reinterpret_cast<float2*>(slab + h * 8 * 128 + ((((j % 4) * 2) ^ res_xor) << 4));
        float2 rr = make_float2(0.f, 0.f);
        if (RES) rr = *rp;
        float r0 = 0.f, r1 = 0.f;
        if (TMA_OUT) {
          // the same values as below, into shared memory: the fp32 sum where its residual was read (no other thread
          // touches that address; RES: its bf16 copy is made from there once the staging chunk is free), the bf16
          // pair into the staging box (rows past M are clipped by the store maps; N is a multiple of 8, so
          // col + 1 < N)
          if (RES) {
            v0 += rr.x;
            v1 += rr.y;
            *rp = make_float2(v0, v1);
          }
          const uint32_t pk = pack_bf16x2(v0, v1);
          if (!RES) *reinterpret_cast<uint32_t*>(stg + h * 8 * 128) = pk;
          r0 = __uint_as_float(pk << 16);
          r1 = __uint_as_float(pk & 0xFFFF0000u);
        } else if (pair) {
          if (RES) {
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
          const float vv[2] = {v0, v1}, res[2] = {rr.x, rr.y};
          float rb[2] = {0.f, 0.f};
          for (int i = 0; i < 2 && col + i < p.N; ++i) {
            float x = vv[i];
            if (RES) x += res[i];
            if (p.out_f32) p.out_f32[o + i] = x;
            const __nv_bfloat16 xb = __float2bfloat16_rn(x);
            if (p.out_bf16) p.out_bf16[o + i] = xb;
            rb[i] = __bfloat162float(xb);
          }
          r0 = rb[0];
          r1 = rb[1];
        }
        if (flags & B200VIT_EPI_STATS) {
          st_sum[h][j / 8] += r0 + r1;
          st_sq[h][j / 8] = fmaf(r0, r0, fmaf(r1, r1, st_sq[h][j / 8]));
        }
      }
      if (RES && j % 8 == 7 && j / 8 < nslab) {
        if constexpr (TMA_OUT) {
          // The previous slab's stores have had this slab's arithmetic to read the chunk and their slab: wait for
          // them, hand that slab back to its loader, then stage this slab's bf16 copy -- rounded from the fp32 sums
          // this thread wrote into the slab, rather than held in registers -- and store the slab and the chunk.
          if (t == 0) {
            tma_store_wait_read<0>();
            if (pend_slab >= 0) mbar_arrive(&empty_bar[pend_slab]);
            pend_slab = -1;
          }
          warpgroup_sync(c);
          if (p.out_bf16)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float2 s = *reinterpret_cast<const float2*>(slab_base + (jj / 4) * L::RES_BOX + res_off +
                                                                  h * 8 * 128 + ((((jj % 4) * 2) ^ res_xor) << 4));
                *reinterpret_cast<uint32_t*>(stg_wg + stg_off + ((jj ^ (lane >> 2)) << 4) + h * 8 * 128) =
                    pack_bf16x2(s.x, s.y);
              }
          fence_proxy_async_smem();
          warpgroup_sync(c);
          if (t == 0) {
            const int c0 = n0 + 64 * (j / 8), row0 = m_blk * BLOCK_M + 64 * c;
            if (row0 < p.M) {
              const uint8_t* half = slab_base + c * 64 * 128;
              if (p.out_f32)
                for (int b = 0; b < 2 && c0 + 32 * b < p.N; ++b)
                  tma_store_2d(&tmF, half + b * L::RES_BOX, c0 + 32 * b, row0);
              if (p.out_bf16) tma_store_2d(&tmO, stg_wg, c0, row0);
            }
            tma_store_commit();
            pend_slab = ring_slab ? stage : STAGES + 2 + (slab_it & 1);
          }
        } else {
          mbar_arrive(&res_empty[slab_it & 1]);
        }
        if (ring_slab) {
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        } else {
          ++slab_it;
        }
      }
    }
    mbar_arrive(&vec_empty[vb]);
    if constexpr (TMA_OUT && !RES) {
      // generic-proxy writes -> visible to the TMA unit, then one thread stores the warpgroup's 64 rows, box by box
      fence_proxy_async_smem();
      warpgroup_sync(c);
      if (t == 0) {
        const int row0 = m_blk * BLOCK_M + 64 * c;
        if (row0 < p.M)
          for (int b = 0; b < BLOCK_N / 64 && n0 + 64 * b < p.N; ++b)
            tma_store_2d(&tmO, stg_wg + b * L::OUT_BOX, n0 + 64 * b, row0);
        tma_store_commit();
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
          // (row[0] + 8 h rather than row[h]: holding row[1] through the epilogue spills at 256 columns)
          float* so = p.stats_out + 2 * (size_t)(row[0] + 8 * h) * p.stats_parts;
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
  if (TMA_OUT && t == 0) tma_store_wait<0>();
}

// test hook 12: BLOCK_N of b200vit_gemm_bf16 -- 0 = auto, 1 = 128, 2 = 256
static std::atomic<int> g_gemm_block_n{0};
void gemm_set_block_n(int v) { g_gemm_block_n = v; }
// test hook 14: 1 = every b200vit_gemm_bf16 launch takes the direct-store epilogue
static std::atomic<int> g_gemm_direct_store{0};
void gemm_set_direct_store(int v) { g_gemm_direct_store = v; }

template <int BLOCK_N, int STAGES, bool PATCH = false, bool RES = false, bool TMA_OUT = false, bool SIG = false,
          int EPI = -1>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmR, const CUtensorMap& tmO,
                       const CUtensorMap& tmF, GemmParams& p, cudaStream_t stream) {
  using L = GemmSmem<BLOCK_N, STAGES, PATCH, RES, TMA_OUT>;
  // 256 x 4 residual with TMA stores (slabs in the ring): 4 x 48 KB ring + 16 KB staging chunk + 1 KB bias + 128 B
  // barriers + 1 KB alignment slack = 215 168 of the 232 448 bytes
  static_assert(L::DYN_BYTES <= 227 * 1024, "gemm: shared memory budget");
  static_assert(!L::BIAS_ONLY || L::DYN_BYTES == 215168, "gemm: 256 x 4 residual TMA-store layout changed");
  auto kern = gemm_bf16_kernel<BLOCK_N, STAGES, PATCH, RES, TMA_OUT, SIG, EPI>;
  B200_ENSURE_SMEM(kern, L::DYN_BYTES);
  if (!p.patch) p.rows_per_tile = BLOCK_M;
  p.num_m_tiles = (p.M + p.rows_per_tile - 1) / p.rows_per_tile;
  p.num_n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  p.num_k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
  p.stats_width = p.N > 128 ? 128 : 64;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, NUM_THREADS, L::DYN_BYTES, stream>>>(tmA, tmB, tmR, tmO, tmF, p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// TMA-store launches with the encoder layer's flag sets -- QKV (bias + LN fold), FC1 (the same + GELU), out-proj and
// FC2 (residual + statistics, with or without a bias) -- run instances compiled for exactly those flags; any other set
// runs the generic instance
template <int BLOCK_N, int STAGES, bool RES>
static int launch_tma_out(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmR,
                          const CUtensorMap& tmO, const CUtensorMap& tmF, GemmParams& p, cudaStream_t stream) {
  constexpr int QKV = B200VIT_EPI_BIAS | B200VIT_EPI_LNFOLD, FC1 = QKV | B200VIT_EPI_GELU;
  constexpr int RES_STATS = B200VIT_EPI_RESIDUAL | B200VIT_EPI_STATS, RES_STATS_BIAS = RES_STATS | B200VIT_EPI_BIAS;
  if constexpr (RES) {
    if (p.flags == RES_STATS_BIAS)
      return launch_gemm<BLOCK_N, STAGES, false, true, true, false, RES_STATS_BIAS>(tmA, tmB, tmR, tmO, tmF, p, stream);
    if (p.flags == RES_STATS)
      return launch_gemm<BLOCK_N, STAGES, false, true, true, false, RES_STATS>(tmA, tmB, tmR, tmO, tmF, p, stream);
  } else {
    if (p.flags == QKV)
      return launch_gemm<BLOCK_N, STAGES, false, false, true, false, QKV>(tmA, tmB, tmR, tmO, tmF, p, stream);
    if (p.flags == FC1)
      return launch_gemm<BLOCK_N, STAGES, false, false, true, false, FC1>(tmA, tmB, tmR, tmO, tmF, p, stream);
  }
  return launch_gemm<BLOCK_N, STAGES, false, RES, true>(tmA, tmB, tmR, tmO, tmF, p, stream);
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
  B200_CHECK_ARG(!(flags & B200VIT_EPI_RESIDUAL) || (ldo & 3) == 0,
                 "gemm: EPI_RESIDUAL needs ldo=%lld to be a multiple of 4 (16-byte rows for TMA)", (long long)ldo);
  B200_CHECK_ARG(!(flags & B200VIT_EPI_LNFOLD) || (ln_sums && col_s && ln_parts >= 1 && ln_parts <= 64),
                 "gemm: EPI_LNFOLD needs ln_sums, col_s and 1 <= ln_parts <= 64");
  B200_CHECK_ARG(!(flags & B200VIT_EPI_STATS) || stats_out, "gemm: EPI_STATS without stats_out");
  B200_CHECK_ARG(!(flags & B200VIT_EPI_RESIDUAL) || !(flags & (B200VIT_EPI_SILU | B200VIT_EPI_SIGMOID)),
                 "gemm: EPI_SILU and EPI_SIGMOID do not combine with EPI_RESIDUAL");
  const int act = flags & (B200VIT_EPI_GELU | B200VIT_EPI_HARDSWISH | B200VIT_EPI_SILU | B200VIT_EPI_SIGMOID);
  B200_CHECK_ARG((act & (act - 1)) == 0,
                 "gemm: EPI_GELU, EPI_HARDSWISH, EPI_SILU and EPI_SIGMOID are exclusive (flags 0x%x)", flags);
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
  p.ln_sums = ln_sums;
  p.ln_parts = ln_parts;
  p.stats_parts = b200vit_stats_parts(N);
  p.ln_inv_dim = 1.0f / (float)K;
  p.ln_eps = ln_eps;
  p.col_s = col_s;
  p.stats_out = stats_out;

  const bool res = (flags & B200VIT_EPI_RESIDUAL) != 0;
  // The TMA-store epilogue takes bf16 outputs and residual launches (fp32 + bf16), with ldo and N multiples of 8 so
  // that every row and its written part are whole 16-byte units (a precaution at N: the store maps clip there anyway).
  // A non-residual fp32 output (off the hot path) has no room for its 128 KB staging tile and stores from the
  // registers, as do patch tiles.  A 256-wide residual tile with TMA stores has room for the bias slice only, so a
  // residual launch with an LN fold runs 128-wide tiles (or, forced wide by test hook 12, stores directly).
  const bool tma_ok = !g_gemm_direct_store.load() && ((ldo | N) & 7) == 0 && (res || !out_f32);
  const bool lnfold = (flags & B200VIT_EPI_LNFOLD) != 0;
  const int force = g_gemm_block_n.load();
  // Residual launches take 256-wide tiles when there is at least one wide tile per SM (fewer would leave SMs idle).
  // Measured on an H100 SXM at 700 W, M = 100 864, N = 768: K 768 (out-proj) 0.42-0.44 ms against 0.48-0.50 at 128
  // columns, K 3072 (FC2) 0.91-0.93 ms against 0.95-0.97.
  const bool res_wide_pays = (long long)((M + BLOCK_M - 1) / BLOCK_M) * ((N + 255) / 256) >= num_sms();
  // SiLU / sigmoid launches (squeeze-excitation over a few pooled rows) take their own 128-wide instances
  const bool sig = (flags & (B200VIT_EPI_SILU | B200VIT_EPI_SIGMOID)) != 0;
  const bool wide = !sig && (force == 0 ? N > 128 && (!(res && tma_ok) || (!lnfold && res_wide_pays)) : force == 2);
  const uint32_t block_n = wide ? 256 : 128;
  const bool tma_out = tma_ok && !(res && wide && lnfold);
  CUtensorMap tmA, tmB, tmR{}, tmO{}, tmF{};
  if (tma_out && out_bf16) {
    const uint64_t dims[2] = {(uint64_t)N, (uint64_t)M};
    const uint64_t strides[1] = {(uint64_t)ldo * 2};
    const uint32_t box[2] = {64, 64};
    int rc = encode_tmap_bf16(&tmO, out_bf16, 2, dims, strides, box);
    if (rc) return rc;
  }
  if (tma_out && res && out_f32) {
    // the residual slab's layout: 32-column boxes (128 B rows, 128B swizzle), 64 rows per consumer warpgroup
    const uint64_t dims[2] = {(uint64_t)N, (uint64_t)M};
    const uint64_t strides[1] = {(uint64_t)ldo * 4};
    const uint32_t box[2] = {32, 64};
    int rc = encode_tmap_f32(&tmF, out_f32, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  if (res) {
    // fp32 residual, 32-column boxes (128 B rows, 128B swizzle) of one tile's 128 rows
    const uint64_t dims[2] = {(uint64_t)N, (uint64_t)M};
    const uint64_t strides[1] = {(uint64_t)ldo * 4};
    const uint32_t box[2] = {32, (uint32_t)BLOCK_M};
    int rc = encode_tmap_f32(&tmR, resid, 2, dims, strides, box, true);
    if (rc) return rc;
  }
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
  if (sig)
    return tma_out ? launch_gemm<128, 5, false, false, true, true>(tmA, tmB, tmR, tmO, tmF, p, st)
                   : launch_gemm<128, 6, false, false, false, true>(tmA, tmB, tmR, tmO, tmF, p, st);
  // residual launches trade ring stages for the two 32 KB residual slabs, TMA-store launches for the staging buffers
  if (tma_out) {
    if (res)
      return wide ? launch_tma_out<256, 4, true>(tmA, tmB, tmR, tmO, tmF, p, st)
                  : launch_tma_out<128, 4, true>(tmA, tmB, tmR, tmO, tmF, p, st);
    return wide ? launch_tma_out<256, 3, false>(tmA, tmB, tmR, tmO, tmF, p, st)
                : launch_tma_out<128, 5, false>(tmA, tmB, tmR, tmO, tmF, p, st);
  }
  if (wide)
    return res ? launch_gemm<256, 3, false, true>(tmA, tmB, tmR, tmO, tmF, p, st)
               : launch_gemm<256, 4>(tmA, tmB, tmR, tmO, tmF, p, st);
  return res ? launch_gemm<128, 4, false, true>(tmA, tmB, tmR, tmO, tmF, p, st)
             : launch_gemm<128, 6>(tmA, tmB, tmR, tmO, tmF, p, st);
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
  B200_CHECK_ARG(head_width_ok(dh), "gemm_headnorm: dim_head=%d not supported by this build (32, 64, 80 or 128)", dh);
  B200_CHECK_ARG(norm_heads > 0 && norm_heads * dh <= N, "gemm_headnorm: %d heads do not fit N=%d", norm_heads, N);
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
  CUtensorMap tmA, tmB, tmR{}, tmO{}, tmF{};
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
  return launch_gemm<256, 4, true>(tmA, tmB, tmR, tmO, tmF, p, reinterpret_cast<cudaStream_t>(stream));
}
