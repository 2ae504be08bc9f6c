// Multi-head softmax attention straight out of the packed QKV buffer, for sm_90a:
//   b200vit_attention          B sequences of N tokens (N <= 512; 128 < N <= 256 at dh 32 / 64 runs the persistent
//                              kernel of attention_short.cu instead, same bits)
//   b200vit_attention_varlen   packed sequences of any length (cu_seqlens), the block-diagonal attention of NaViT and
//                              the long-sequence path of ViT
// One CTA = one 128-row query tile of one (sequence, head): two warpgroups of 64 query rows each.  Thread 0 loads the
// Q tile and the K / V blocks of KB keys with TMA into a two-stage ring of 128B-swizzled shared memory (mbarrier
// complete_tx; a stage is reloaded once both warpgroups have released it).  Per key block each warpgroup computes
// S = Q K^T with wgmma (both operands in shared memory), runs an online softmax in fp32 on the accumulator registers
// and accumulates O += P V with wgmma, P (bf16) taken from registers as the A operand and V read as the transposed
// (MN-major) B operand.  dh = 32, 64, 80 or 128: a head is split into 64-wide (128B swizzle) and 16-wide (32B swizzle)
// slabs (AttnSmem).  Keys of a block beyond the sequence get probability 0, and their V rows are zero, so that a NaN or
// Inf in one sequence cannot reach another through 0 x NaN in O += P V: the fixed-length kernel reads Q, K and V
// through 3-D tensor maps (column, token, sequence), which zero-fill past the end of each sequence; the varlen kernel
// reads the packed rows through 2-D maps and zeroes the V rows beyond the sequence of its last key block in shared
// memory.
// MASK_SELF instances (b200vit_attention_ex / _varlen_ex with B200VIT_ATTN_MASK_SELF) also give key i of query i
// probability 0 -- LSA, vit_for_small_dataset.py:53-57 -- except in a sequence of one token, where the reference's
// -finfo.max fill leaves that token's own key with weight 1.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int ATT_QROWS = 128;
constexpr int ATT_THREADS = 256;

struct AttnParams {
  __nv_bfloat16* out;
  int N;                      // fixed-length mode: tokens per sequence (grid.z = sequence)
  const int32_t* cu_seqlens;  // varlen mode: [num_seqs + 1] token offsets, tile_prefix: 128-row tiles before s
  const int32_t* tile_prefix;
  int num_seqs;
  int H, I;                   // heads, H * dh
  float scale_log2e;
};

// A head of DH columns is DH / 64 slabs 64 columns wide (128B swizzle) followed by (DH % 64) / 16 slabs 16 columns
// wide (32B swizzle): dh 32 = 2 x 16, 64 = 64, 80 = 64 + 16, 128 = 2 x 64.  Shared memory: Q64[N64] | Q16[N16], then
// per stage K64[N64] | V64[N64] | K16[N16] | V16[N16].
constexpr int KB = 64;  // keys per block
template <int DH>
struct AttnSmem {
  static constexpr int N64 = DH / 64;
  static constexpr int N16 = (DH % 64) / 16;
  static_assert(N64 * 64 + N16 * 16 == DH, "dim_head must be a multiple of 16");
  static constexpr int Q64 = ATT_QROWS * 128;        // one 64-column slab of Q
  static constexpr int Q16 = ATT_QROWS * 32;         // one 16-column slab of Q
  static constexpr int KV64 = KB * 128;
  static constexpr int KV16 = KB * 32;
  static constexpr int K16_OFF = 2 * N64 * KV64;     // within a stage
  static constexpr int V16_OFF = K16_OFF + N16 * KV16;
  static constexpr int STAGE = 2 * (N64 * KV64 + N16 * KV16);
  static constexpr int STAGE_OFF = N64 * Q64 + N16 * Q16;
  static constexpr int BAR_OFF = STAGE_OFF + 2 * STAGE;
  static constexpr int BYTES = BAR_OFF + 5 * 8 + 1024;  // full[2], empty[2], q; slack for 1024B alignment
};

// CTAs per SM the register budget is planned for (ptxas -v: no spills at these bounds).  dh 160 = 2 x 64 + 2 x 16
// (varlen only, the one head of a T2T-ViT soft split up to 160 wide): 40 KB of Q and two 40 KB K / V stages.
constexpr int att_min_blocks(int dh) { return dh == 64 || dh == 32 ? 2 : 1; }

template <int DH, bool VARLEN, bool MASK_SELF>
__global__ void __launch_bounds__(ATT_THREADS, att_min_blocks(DH))
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                 const __grid_constant__ CUtensorMap tmQ16, const __grid_constant__ CUtensorMap tmKV16,
                 const AttnParams p) {
  using L = AttnSmem<DH>;
  constexpr int N64 = L::N64, N16 = L::N16;
  constexpr int NS = KB / 2;  // score accumulators per thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty = full + 2;
  uint64_t* qbar = full + 4;

  const int h = blockIdx.y;
  int seq_start, len, q0;
  if (VARLEN) {
    const int tile = blockIdx.x;
    int lo = 0, hi = p.num_seqs - 1;  // last s with tile_prefix[s] <= tile
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (p.tile_prefix[mid] <= tile) lo = mid;
      else hi = mid - 1;
    }
    seq_start = p.cu_seqlens[lo];
    len = p.cu_seqlens[lo + 1] - seq_start;
    q0 = (tile - p.tile_prefix[lo]) * ATT_QROWS;
  } else {
    seq_start = blockIdx.z * p.N;
    len = p.N;
    q0 = blockIdx.x * ATT_QROWS;
  }
  const int nblocks = (len + KB - 1) / KB;
  const int colq = h * DH, colk = p.I + h * DH, colv = 2 * p.I + h * DH;
  const int tid = threadIdx.x;
  const int wg = tid >> 7, t = tid & 127, warp = t >> 5, lane = t & 31;

  // rows from token `tok` of this sequence: packed rows (varlen), or the (column, token, sequence) view
  auto load = [&](void* dst, const CUtensorMap* tm, uint64_t* bar, int col, int tok) {
    if (VARLEN) tma_load_2d(dst, tm, bar, col, seq_start + tok);
    else tma_load_3d(dst, tm, bar, col, tok, blockIdx.z);
  };
  auto issue_kv = [&](int blk) {
    const int st = blk & 1;
    uint8_t* sb = smem + L::STAGE_OFF + st * L::STAGE;
    const int tok = blk * KB;
    mbar_arrive_expect_tx(&full[st], L::STAGE);
#pragma unroll
    for (int c = 0; c < N64; ++c) {
      load(sb + c * L::KV64, &tmKV, &full[st], colk + 64 * c, tok);
      load(sb + (N64 + c) * L::KV64, &tmKV, &full[st], colv + 64 * c, tok);
    }
#pragma unroll
    for (int c = 0; c < N16; ++c) {
      load(sb + L::K16_OFF + c * L::KV16, &tmKV16, &full[st], colk + 64 * N64 + 16 * c, tok);
      load(sb + L::V16_OFF + c * L::KV16, &tmKV16, &full[st], colv + 64 * N64 + 16 * c, tok);
    }
  };

  if (tid == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrive per warpgroup
    }
    mbar_init(qbar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(qbar, L::STAGE_OFF);
#pragma unroll
    for (int c = 0; c < N64; ++c) load(smem + c * L::Q64, &tmQ, qbar, colq + 64 * c, q0);
#pragma unroll
    for (int c = 0; c < N16; ++c) load(smem + N64 * L::Q64 + c * L::Q16, &tmQ16, qbar, colq + 64 * N64 + 16 * c, q0);
    issue_kv(0);
    if (nblocks > 1) issue_kv(1);
  }

  // per-slab output accumulators (an array of extent 1 stands in for an absent kind; the compiler drops it)
  float o[N64 > 0 ? N64 : 1][32], o16[N16 > 0 ? N16 : 1][8];
#pragma unroll
  for (int c = 0; c < N64; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
#pragma unroll
  for (int c = 0; c < N16; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) o16[c][i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t qa = smem_u32(smem) + wg * 64 * 128;
  const uint32_t qa16 = smem_u32(smem + N64 * L::Q64) + wg * 64 * 32;
  // a length-1 sequence keeps its only key (see above), so for len >= 2 every row has a valid key in block 0 (keys 0 and
  // 1) and m is finite from there on: no -inf - -inf
  const bool mask_self = MASK_SELF && len > 1;
  mbar_wait(qbar, 0);

  for (int kb = 0; kb < nblocks; ++kb) {
    const int st = kb & 1;
    const uint32_t ph = (kb >> 1) & 1;
    mbar_wait(&full[st], ph);
    const uint32_t sb = smem_u32(smem + L::STAGE_OFF + st * L::STAGE);
    if (VARLEN && kb == nblocks - 1 && len % KB != 0) {
      // the last block's rows beyond the sequence are the next sequence's tokens: zero their V (P is 0 there, but
      // 0 x NaN is NaN), then make the writes visible to the wgmma reads of both warpgroups
      const int r0 = len - kb * KB;
      uint8_t* stage = smem + L::STAGE_OFF + st * L::STAGE;
      const uint4 z = make_uint4(0u, 0u, 0u, 0u);
      // the swizzles permute 16-byte chunks within a row: row r of a slab is bytes [128 r, 128 r + 128) (64 wide) or
      // [32 r, 32 r + 32) (16 wide)
#pragma unroll
      for (int c = 0; c < N64; ++c) {
        uint4* sl = reinterpret_cast<uint4*>(stage + (N64 + c) * L::KV64);
        for (int i = r0 * 8 + tid; i < KB * 8; i += ATT_THREADS) sl[i] = z;
      }
#pragma unroll
      for (int c = 0; c < N16; ++c) {
        uint4* sl = reinterpret_cast<uint4*>(stage + L::V16_OFF + c * L::KV16);
        for (int i = r0 * 2 + tid; i < KB * 2; i += ATT_THREADS) sl[i] = z;
      }
      fence_proxy_async_smem();
      __syncthreads();
    }

    // S = Q K^T (64 rows x KB keys per warpgroup): one k16 step per 16 columns, the 64-wide slabs first
    float s[NS];
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < N64; ++c)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t ad = make_wgmma_desc(qa + c * L::Q64, 1024, WGMMA_SW128) + 2 * k;
        const uint64_t bd = make_wgmma_desc(sb + c * L::KV64, 1024, WGMMA_SW128) + 2 * k;
        wgmma_m64n64k16(s, ad, bd, c != 0 || k != 0);
      }
#pragma unroll
    for (int c = 0; c < N16; ++c) {
      const uint64_t ad = make_wgmma_desc(qa16 + c * L::Q16, 256, WGMMA_SW32);
      const uint64_t bd = make_wgmma_desc(sb + L::K16_OFF + c * L::KV16, 256, WGMMA_SW32);
      wgmma_m64n64k16(s, ad, bd, N64 != 0 || c != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);

    // online softmax (log2 units); s[4j + e]: row 16 warp + lane/4 + 8 (e >> 1), key 8 j + 2 (lane % 4) + (e & 1)
    const int key0 = kb * KB + 2 * (lane & 3);
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int j = 0; j < KB / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = key0 + j * 8 + (e & 1);
        bool valid = key < len;
        if constexpr (MASK_SELF)  // query index within the sequence of accumulator row e >> 1
          valid = valid && !(mask_self && key == q0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * (e >> 1));
        s[4 * j + e] = valid ? s[4 * j + e] * p.scale_log2e : -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * j + e]);
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float corr = fast_ex2(m[r] - mx[r]);  // m = -inf on the first block: exp2(-inf) = 0
      l[r] *= corr;
#pragma unroll
      for (int c = 0; c < N64; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[c][4 * i + 2 * r] *= corr;
          o[c][4 * i + 2 * r + 1] *= corr;
        }
#pragma unroll
      for (int c = 0; c < N16; ++c)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          o16[c][4 * i + 2 * r] *= corr;
          o16[c][4 * i + 2 * r + 1] *= corr;
        }
      m[r] = mx[r];
    }
#pragma unroll
    for (int j = 0; j < KB / 8; ++j) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float e0 = fast_ex2(s[4 * j + 2 * r] - m[r]), e1 = fast_ex2(s[4 * j + 2 * r + 1] - m[r]);
        s[4 * j + 2 * r] = e0;
        s[4 * j + 2 * r + 1] = e1;
        l[r] += e0 + e1;
      }
    }

    // O += P V: the score accumulators of 16 keys are the A fragment of one k-step (bf16); one MMA per slab
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KB / 16; ++kk) {
      const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                             pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
#pragma unroll
      for (int c = 0; c < N64; ++c)
        wgmma_m64n64k16_rs_tb(o[c], a,
                              make_wgmma_desc_lbo(sb + (N64 + c) * L::KV64 + kk * 2048, 1024, 1024, WGMMA_SW128));
#pragma unroll
      for (int c = 0; c < N16; ++c)
        wgmma_m64n16k16_rs_tb(o16[c], a,
                              make_wgmma_desc_lbo(sb + L::V16_OFF + c * L::KV16 + kk * 512, 256, 256, WGMMA_SW32));
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < N64; ++c) fence_regs(o[c]);
#pragma unroll
    for (int c = 0; c < N16; ++c) fence_regs(o16[c]);
    if (t == 0) mbar_arrive(&empty[st]);
    if (tid == 0 && kb + 2 < nblocks) {
      mbar_wait(&empty[st], ph);  // both warpgroups are done with this stage
      issue_kv(kb + 2);
    }
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    l[r] = 1.0f / l[r];
  }
  const int qr = q0 + wg * 64 + warp * 16 + (lane >> 2);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = qr + 8 * r;
    if (row >= len) continue;
    __nv_bfloat16* op = p.out + (long long)(seq_start + row) * p.I + h * DH + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < N64; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(op + 64 * c + j * 8) =
            pack_bf16x2(o[c][4 * j + 2 * r] * l[r], o[c][4 * j + 2 * r + 1] * l[r]);
#pragma unroll
    for (int c = 0; c < N16; ++c)
#pragma unroll
      for (int j = 0; j < 2; ++j)
        *reinterpret_cast<uint32_t*>(op + 64 * N64 + 16 * c + j * 8) =
            pack_bf16x2(o16[c][4 * j + 2 * r] * l[r], o16[c][4 * j + 2 * r + 1] * l[r]);
  }
}

// Tensor maps over qkv[T, 3 I] (varlen) or its [B][N][3 I] view (fixed length, T = B N): 64-column boxes (128B swizzle)
// of 128 query rows / KB key rows for the 64-wide slabs, and the same with 16 columns (32B swizzle) for the 16-wide
// ones.  A kind the head does not use gets a copy of the other (never read).
template <int DH, bool VARLEN, bool MASK_SELF>
static int launch_attention_t(const void* qkv, int T, const AttnParams& p, dim3 grid, cudaStream_t stream) {
  using L = AttnSmem<DH>;
  CUtensorMap tm[4];
  const int rank = VARLEN ? 2 : 3;
  const uint64_t ld = (uint64_t)3 * p.I;
  const uint64_t dims[3] = {ld, (uint64_t)(VARLEN ? T : p.N), (uint64_t)(VARLEN ? 1 : T / p.N)};
  const uint64_t strides[2] = {ld * 2, ld * 2 * (VARLEN ? T : p.N)};
  const uint32_t qbox[3] = {64, ATT_QROWS, 1}, kvbox[3] = {64, KB, 1}, qbox16[3] = {16, ATT_QROWS, 1},
                 kvbox16[3] = {16, KB, 1};
  int rc = 0;
  if (L::N64) rc = encode_tmap_bf16(&tm[0], qkv, rank, dims, strides, qbox);
  if (!rc && L::N64) rc = encode_tmap_bf16(&tm[1], qkv, rank, dims, strides, kvbox);
  if (!rc && L::N16) rc = encode_tmap_bf16_sw(&tm[2], qkv, rank, dims, strides, qbox16, 32);
  if (!rc && L::N16) rc = encode_tmap_bf16_sw(&tm[3], qkv, rank, dims, strides, kvbox16, 32);
  if (rc) return rc;
  if (!L::N16) tm[2] = tm[0], tm[3] = tm[1];
  if (!L::N64) tm[0] = tm[2], tm[1] = tm[3];
  auto kern = attention_kernel<DH, VARLEN, MASK_SELF>;
  B200_ENSURE_SMEM(kern, L::BYTES);
  kern<<<grid, ATT_THREADS, L::BYTES, stream>>>(tm[0], tm[1], tm[2], tm[3], p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

template <int DH, bool VARLEN>
static int launch_attention_dh(const void* qkv, int T, const AttnParams& p, bool mask_self, dim3 grid,
                               cudaStream_t st) {
  return mask_self ? launch_attention_t<DH, VARLEN, true>(qkv, T, p, grid, st)
                   : launch_attention_t<DH, VARLEN, false>(qkv, T, p, grid, st);
}

// one instance per width of head_width_ok() (dh 96 = 64 + 2 x 16 would fall out of the same slab scheme), and the
// varlen kernel at dh 160 without self-masking (varlen_head_width_ok)
template <bool VARLEN>
static int launch_attention(const void* qkv, int T, const AttnParams& p, int dh, bool mask_self, dim3 grid,
                            cudaStream_t st) {
  if constexpr (VARLEN)
    if (dh == 160) return launch_attention_t<160, true, false>(qkv, T, p, grid, st);
  switch (dh) {
    case 32: return launch_attention_dh<32, VARLEN>(qkv, T, p, mask_self, grid, st);
    case 80: return launch_attention_dh<80, VARLEN>(qkv, T, p, mask_self, grid, st);
    case 128: return launch_attention_dh<128, VARLEN>(qkv, T, p, mask_self, grid, st);
    default: return launch_attention_dh<64, VARLEN>(qkv, T, p, mask_self, grid, st);
  }
}

// test hook (include/b200vit.h)
static std::atomic<int> g_attn_tiled{0};  // key 15

}  // namespace b200

using namespace b200;

extern "C" int b200vit_debug_set(int key, int value) {
  switch (key) {
    case 12: gemm_set_block_n(value); return 0;
    case 14: gemm_set_direct_store(value); return 0;
    case 15: g_attn_tiled = value; return 0;
    default: return B200VIT_ERR_INVALID;
  }
}

extern "C" int b200vit_attention(const void* qkv, void* out, int B, int N, int H, int dh, float scale, void* stream) {
  return b200vit_attention_ex(qkv, out, B, N, H, dh, scale, 0, stream);
}

extern "C" int b200vit_attention_ex(const void* qkv, void* out, int B, int N, int H, int dh, float scale, int flags,
                                    void* stream) {
  B200_CHECK_ARG(qkv && out, "attention: null pointer");
  B200_CHECK_ARG(B > 0 && N > 0 && H > 0, "attention: bad shape B=%d N=%d H=%d", B, N, H);
  B200_CHECK_ARG(head_width_ok(dh), "attention: dim_head=%d not supported by this build (32, 64, 80 or 128)", dh);
  B200_CHECK_ARG(N <= 512, "attention: N=%d > 512 goes through b200vit_attention_varlen", N);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "attention: pointers must be 16-byte aligned");
  B200_CHECK_ARG(B <= 65535, "attention: B=%d exceeds the grid", B);
  B200_CHECK_ARG((flags & ~B200VIT_ATTN_MASK_SELF) == 0, "attention: unknown flags 0x%x", flags);
  // 129 to 256 tokens: the persistent kernel of attention_short.cu, which gives the same bits.  The self-masked
  // instances exist in this file only, and test hook 15 asks for this file's kernel.
  const bool tiled_only = (flags & B200VIT_ATTN_MASK_SELF) || g_attn_tiled.load() != 0;
  if (!tiled_only && attention_short_ok(N, dh))
    return attention_short(qkv, out, B, N, H, dh, scale * 1.4426950408889634f, reinterpret_cast<cudaStream_t>(stream));
  AttnParams p{};
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.N = N;
  p.H = H;
  p.I = H * dh;
  p.scale_log2e = scale * 1.4426950408889634f;
  const dim3 grid((N + ATT_QROWS - 1) / ATT_QROWS, H, B);
  return launch_attention<false>(qkv, B * N, p, dh, (flags & B200VIT_ATTN_MASK_SELF) != 0, grid,
                                 reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b200vit_attention_varlen(const void* qkv, void* out, const int32_t* cu_seqlens_dev,
                                        const int32_t* tile_prefix_dev, int num_seqs, int total_tokens, int total_tiles,
                                        int H, int dh, float scale, void* stream) {
  return b200vit_attention_varlen_ex(qkv, out, cu_seqlens_dev, tile_prefix_dev, num_seqs, total_tokens, total_tiles, H,
                                     dh, scale, 0, stream);
}

extern "C" int b200vit_attention_varlen_ex(const void* qkv, void* out, const int32_t* cu_seqlens_dev,
                                           const int32_t* tile_prefix_dev, int num_seqs, int total_tokens,
                                           int total_tiles, int H, int dh, float scale, int flags, void* stream) {
  B200_CHECK_ARG(qkv && out && cu_seqlens_dev && tile_prefix_dev, "attention_varlen: null pointer");
  B200_CHECK_ARG(num_seqs > 0 && total_tokens > 0 && total_tiles > 0 && H > 0, "attention_varlen: bad shape");
  B200_CHECK_ARG(head_width_ok(dh) || (dh == 160 && !(flags & B200VIT_ATTN_MASK_SELF)),
                 "attention_varlen: dim_head=%d not supported by this build (32, 64, 80 or 128), nor 160 with "
                 "B200VIT_ATTN_MASK_SELF", dh);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "attention_varlen: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535, "attention_varlen: H=%d exceeds the grid", H);
  B200_CHECK_ARG((flags & ~B200VIT_ATTN_MASK_SELF) == 0, "attention_varlen: unknown flags 0x%x", flags);
  AttnParams p{};
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.cu_seqlens = cu_seqlens_dev;
  p.tile_prefix = tile_prefix_dev;
  p.num_seqs = num_seqs;
  p.H = H;
  p.I = H * dh;
  p.scale_log2e = scale * 1.4426950408889634f;
  const dim3 grid(total_tiles, H, 1);
  return launch_attention<true>(qkv, total_tokens, p, dh, (flags & B200VIT_ATTN_MASK_SELF) != 0, grid,
                                reinterpret_cast<cudaStream_t>(stream));
}
