// Softmax attention for B sequences of N tokens with 128 < N <= 256 and dh = 32 or 64: the bits of attention_kernel
// (attention.cu), from a persistent kernel that stages every head once.
//
// One CTA per SM loops over (sequence, head) items.  Four consumer warpgroups own 64 query rows each (4 x 64 >= N; a
// warpgroup whose rows all lie past N leaves at once and is not counted on any barrier) and one producer thread feeds
// them with TMA.  An item's Q, K and V -- 3 x 256 rows x dh, 96 KB at dh 64 -- are resident in 128B / 32B-swizzled
// shared memory, and there are two such buffers, so the producer loads item i + 1 while the consumers work on item i.
// Every 64-key block of K and V has a full barrier of its own: a warpgroup starts on block 0 as soon as it has landed.
// Q, K and V come through the 3-D (column, token, sequence) view of the packed buffer, whose zero fill past the end of
// each sequence keeps one sequence's NaN / Inf out of another's (see attention.cu).
//
// Per key block a warpgroup does what attention_kernel<DH, 64> does, in the same order: S = Q K^T by wgmma from shared
// memory, scale, mask, running max, ex2, bf16 P from registers, O += P V with V as the transposed operand.  The one
// difference is that the last block runs at its real width rounded up to 16 keys (n16 / n32 / n48 for S, fewer k16
// steps for P V) instead of 64.  The dropped keys had probability exactly 0 and did not move the running max, so the
// output is bit-identical; N = 197 works on 208 keys per row instead of 256.
//
// A finished warpgroup writes its 64 x dh bf16 block over its own Q rows, which nothing reads any more, and one thread
// stores them with TMA through a 3-D map of `out`, which clips rows past N.  The buffer goes back to the producer once
// every warpgroup's store has read its rows.
//
// dh 80 and 128 do not fit two resident items (2 x 120 KB, 2 x 192 KB) and stay with attention_kernel, as do the
// self-masked launches.  attention_short_ok() is the test; b200vit_attention_ex dispatches on it.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int SH_ROWS = 256;            // tokens a buffer holds
constexpr int SH_KB = 64;               // keys per block
constexpr int SH_WGS = SH_ROWS / 64;    // consumer warpgroups
constexpr int SH_THREADS = SH_WGS * 128 + 32;

struct ShortParams {
  int N, H, items;  // items = B * H
  float scale_log2e;
};

// The slab scheme of AttnSmem (attention.cu) over 256 rows: a buffer is Q | K | V, each N64 slabs of 256 x 128 B
// followed by N16 slabs of 256 x 32 B.  Barriers: qfull[2], kvfull[2][4], empty[2].
template <int DH>
struct ShortSmem {
  static constexpr int N64 = DH / 64;
  static constexpr int N16 = (DH % 64) / 16;
  static constexpr int SLAB64 = SH_ROWS * 128;
  static constexpr int SLAB16 = SH_ROWS * 32;
  static constexpr int MAT = N64 * SLAB64 + N16 * SLAB16;  // one of Q, K, V
  static constexpr int S16_OFF = N64 * SLAB64;             // the 16-wide slabs within it
  static constexpr int ITEM = 3 * MAT;
  static constexpr int BAR_OFF = 2 * ITEM;
  static constexpr int NBARS = 2 + 2 * SH_WGS + 2;
  static constexpr int BYTES = BAR_OFF + NBARS * 8 + 1024;  // slack for 1024B alignment
  static constexpr int ROW_BYTES = DH * 2;
  static_assert(BYTES <= 227 * 1024, "two resident items must fit in shared memory");
};

template <int W>
__device__ __forceinline__ void wgmma_s(float (&s)[W / 2], uint64_t ad, uint64_t bd, uint32_t scale_d) {
  if constexpr (W == 16) wgmma_m64n16k16(s, ad, bd, scale_d);
  else if constexpr (W == 32) wgmma_m64n32k16(s, ad, bd, scale_d);
  else if constexpr (W == 48) wgmma_m64n48k16(s, ad, bd, scale_d);
  else wgmma_m64n64k16(s, ad, bd, scale_d);
}

// One block of W keys starting at key `kbase` for one warpgroup: the per-block body of attention_kernel.  qa / qa16:
// the warpgroup's Q rows in the 64- and 16-wide slabs; ka / ka16 / va / va16: row `kbase` of K and V likewise.
// MASK = false is for a block that lies within the sequence: every key is valid, so the comparison with `len` and
// the select go; the product is rounded on its own (__fmul_rn) as it is where the select follows it.
template <int DH, int W, bool MASK>
__device__ __forceinline__ void short_block(uint32_t qa, uint32_t qa16, uint32_t ka, uint32_t ka16, uint32_t va,
                                            uint32_t va16, int kbase, int len, float scale_log2e, int lane,
                                            float (&o)[DH / 64 > 0 ? DH / 64 : 1][32],
                                            float (&o16)[(DH % 64) / 16 > 0 ? (DH % 64) / 16 : 1][8], float (&m)[2],
                                            float (&l)[2]) {
  using L = ShortSmem<DH>;
  constexpr int N64 = L::N64, N16 = L::N16;
  float s[W / 2];
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < N64; ++c)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t ad = make_wgmma_desc(qa + c * L::SLAB64, 1024, WGMMA_SW128) + 2 * k;
      const uint64_t bd = make_wgmma_desc(ka + c * L::SLAB64, 1024, WGMMA_SW128) + 2 * k;
      wgmma_s<W>(s, ad, bd, c != 0 || k != 0);
    }
#pragma unroll
  for (int c = 0; c < N16; ++c) {
    const uint64_t ad = make_wgmma_desc(qa16 + c * L::SLAB16, 256, WGMMA_SW32);
    const uint64_t bd = make_wgmma_desc(ka16 + c * L::SLAB16, 256, WGMMA_SW32);
    wgmma_s<W>(s, ad, bd, N64 != 0 || c != 0);
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);

  // online softmax (log2 units); s[4j + e]: row 16 warp + lane/4 + 8 (e >> 1), key 8 j + 2 (lane % 4) + (e & 1)
  const int key0 = kbase + 2 * (lane & 3);
  float mx[2] = {m[0], m[1]};
#pragma unroll
  for (int j = 0; j < W / 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int key = key0 + j * 8 + (e & 1);
      s[4 * j + e] = !MASK || key < len ? __fmul_rn(s[4 * j + e], scale_log2e) : -INFINITY;
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
  for (int j = 0; j < W / 8; ++j)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float e0 = fast_ex2(s[4 * j + 2 * r] - m[r]), e1 = fast_ex2(s[4 * j + 2 * r + 1] - m[r]);
      s[4 * j + 2 * r] = e0;
      s[4 * j + 2 * r + 1] = e1;
      l[r] += e0 + e1;
    }

  // O += P V: the score accumulators of 16 keys are the A fragment of one k-step (bf16); one MMA per slab
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < W / 16; ++kk) {
    const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                           pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
#pragma unroll
    for (int c = 0; c < N64; ++c)
      wgmma_m64n64k16_rs_tb(o[c], a, make_wgmma_desc_lbo(va + c * L::SLAB64 + kk * 2048, 1024, 1024, WGMMA_SW128));
#pragma unroll
    for (int c = 0; c < N16; ++c)
      wgmma_m64n16k16_rs_tb(o16[c], a, make_wgmma_desc_lbo(va16 + c * L::SLAB16 + kk * 512, 256, 256, WGMMA_SW32));
  }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < N64; ++c) fence_regs(o[c]);
#pragma unroll
  for (int c = 0; c < N16; ++c) fence_regs(o16[c]);
}

// tmKV / tmKV16: 64-row boxes of 64 / 16 columns of qkv (Q rows are read through them too); tmO / tmO16: the same
// boxes of out, 128B-swizzled / unswizzled.
template <int DH>
__global__ void __launch_bounds__(SH_THREADS, 1)
attention_short_kernel(const __grid_constant__ CUtensorMap tmKV, const __grid_constant__ CUtensorMap tmKV16,
                       const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmO16,
                       const ShortParams p) {
  using L = ShortSmem<DH>;
  constexpr int N64 = L::N64, N16 = L::N16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* qfull = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);  // [2]
  uint64_t* kvfull = qfull + 2;                                      // [2][SH_WGS]
  uint64_t* empty = kvfull + 2 * SH_WGS;                             // [2]

  const int tid = threadIdx.x;
  const int len = p.N;
  const int nblocks = (len + SH_KB - 1) / SH_KB;  // key blocks = warpgroups with rows: 3 or 4
  const int I = p.H * DH;

  if (tid == 0) {
    if (N64) tma_prefetch_desc(&tmKV), tma_prefetch_desc(&tmO);
    if (N16) tma_prefetch_desc(&tmKV16), tma_prefetch_desc(&tmO16);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&qfull[i], 1);
      for (int j = 0; j < SH_WGS; ++j) mbar_init(&kvfull[i * SH_WGS + j], 1);
      mbar_init(&empty[i], nblocks);  // one arrive per warpgroup that has rows
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (__shfl_sync(0xffffffffu, tid >> 7, 0) == SH_WGS) {
    // ---------------------------------------------------------------------------------------------- producer
    if (tid != SH_WGS * 128) return;
    int it = 0;
    for (int item = blockIdx.x; item < p.items; item += gridDim.x, ++it) {
      const int buf = it & 1;
      if (it >= 2) mbar_wait(&empty[buf], ((it >> 1) - 1) & 1);  // every store of the item before has read its rows
      const int b = item / p.H, h = item - b * p.H;
      uint8_t* base = smem + buf * L::ITEM;
      // rows [tok, tok + 64) of matrix `mat` (0 = Q, 1 = K, 2 = V) of this head
      auto load = [&](int mat, int tok, uint64_t* bar) {
        uint8_t* dst = base + mat * L::MAT;
        const int col = mat * I + h * DH;
#pragma unroll
        for (int c = 0; c < N64; ++c) tma_load_3d(dst + c * L::SLAB64 + tok * 128, &tmKV, bar, col + 64 * c, tok, b);
#pragma unroll
        for (int c = 0; c < N16; ++c)
          tma_load_3d(dst + L::S16_OFF + c * L::SLAB16 + tok * 32, &tmKV16, bar, col + 64 * N64 + 16 * c, tok, b);
      };
      mbar_arrive_expect_tx(&qfull[buf], nblocks * SH_KB * L::ROW_BYTES);
      mbar_arrive_expect_tx(&kvfull[buf * SH_WGS], 2 * SH_KB * L::ROW_BYTES);
      load(0, 0, &qfull[buf]);
      load(1, 0, &kvfull[buf * SH_WGS]);
      load(2, 0, &kvfull[buf * SH_WGS]);
      for (int w = 1; w < nblocks; ++w) load(0, w * SH_KB, &qfull[buf]);
      for (int kb = 1; kb < nblocks; ++kb) {
        mbar_arrive_expect_tx(&kvfull[buf * SH_WGS + kb], 2 * SH_KB * L::ROW_BYTES);
        load(1, kb * SH_KB, &kvfull[buf * SH_WGS + kb]);
        load(2, kb * SH_KB, &kvfull[buf * SH_WGS + kb]);
      }
    }
    return;
  }

  // ------------------------------------------------------------------------------------------------ consumers
  // the warpgroup index through a shuffle, so that the compiler knows it to be the same across the warp: with wgmma
  // under a branch it takes to be divergent, it waits for every MMA before it issues the next
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0), t = tid & 127, warp = t >> 5, lane = t & 31;
  if (wg * 64 >= len) return;
  // blocks that lie within the sequence, then the last one at its real width rounded up to 16 keys
  const int nfull = len / SH_KB;
  const int tail_w = ((len - 1) % SH_KB) / 16 * 16 + 16;
  const int row = warp * 16 + (lane >> 2);  // + 8 r: this thread's two rows within the warpgroup

  int it = 0;
  for (int item = blockIdx.x; item < p.items; item += gridDim.x, ++it) {
    const int buf = it & 1;
    const uint32_t ph = (it >> 1) & 1;
    const int b = item / p.H, h = item - b * p.H;
    const uint32_t sq = smem_u32(smem + buf * L::ITEM), sk = sq + L::MAT, sv = sk + L::MAT;
    const uint32_t qa = sq + wg * 64 * 128, qa16 = sq + L::S16_OFF + wg * 64 * 32;

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

    mbar_wait(&qfull[buf], ph);
    for (int kb = 0; kb < nfull; ++kb) {
      mbar_wait(&kvfull[buf * SH_WGS + kb], ph);
      short_block<DH, 64, false>(qa, qa16, sk + kb * 64 * 128, sk + L::S16_OFF + kb * 64 * 32, sv + kb * 64 * 128,
                          sv + L::S16_OFF + kb * 64 * 32, kb * SH_KB, len, p.scale_log2e, lane, o, o16, m, l);
    }
    if (nfull < nblocks) {
      const int kb = nfull;
      mbar_wait(&kvfull[buf * SH_WGS + kb], ph);
      const uint32_t ka = sk + kb * 64 * 128, ka16 = sk + L::S16_OFF + kb * 64 * 32;
      const uint32_t va = sv + kb * 64 * 128, va16 = sv + L::S16_OFF + kb * 64 * 32;
      if (tail_w == 16)
        short_block<DH, 16, true>(qa, qa16, ka, ka16, va, va16, kb * SH_KB, len, p.scale_log2e, lane, o, o16, m, l);
      else if (tail_w == 32)
        short_block<DH, 32, true>(qa, qa16, ka, ka16, va, va16, kb * SH_KB, len, p.scale_log2e, lane, o, o16, m, l);
      else if (tail_w == 48)
        short_block<DH, 48, true>(qa, qa16, ka, ka16, va, va16, kb * SH_KB, len, p.scale_log2e, lane, o, o16, m, l);
      else
        short_block<DH, 64, true>(qa, qa16, ka, ka16, va, va16, kb * SH_KB, len, p.scale_log2e, lane, o, o16, m, l);
    }

#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
      l[r] = 1.0f / l[r];
    }
    // The warpgroup's Q rows have been read for the last time: its output block takes their place, 64-wide slabs in
    // the 128B swizzle of tmO (16-byte chunk j of row r at chunk j ^ (r % 8)), 16-wide slabs as plain 32-byte rows.
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const uint32_t d64 = qa + (row + 8 * r) * 128 + 4 * (lane & 3);
      const uint32_t d16 = qa16 + (row + 8 * r) * 32 + 4 * (lane & 3);
#pragma unroll
      for (int c = 0; c < N64; ++c)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          sts_b32(d64 + c * L::SLAB64 + ((j ^ (lane >> 2)) << 4),
                  pack_bf16x2(o[c][4 * j + 2 * r] * l[r], o[c][4 * j + 2 * r + 1] * l[r]));
#pragma unroll
      for (int c = 0; c < N16; ++c)
#pragma unroll
        for (int j = 0; j < 2; ++j)
          sts_b32(d16 + c * L::SLAB16 + (j << 4),
                  pack_bf16x2(o16[c][4 * j + 2 * r] * l[r], o16[c][4 * j + 2 * r + 1] * l[r]));
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the TMA unit
    asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory");
    if (t == 0) {
      const uint8_t* src = smem + buf * L::ITEM;
#pragma unroll
      for (int c = 0; c < N64; ++c)
        tma_store_3d(&tmO, src + c * L::SLAB64 + wg * 64 * 128, h * DH + 64 * c, wg * 64, b);
#pragma unroll
      for (int c = 0; c < N16; ++c)
        tma_store_3d(&tmO16, src + L::S16_OFF + c * L::SLAB16 + wg * 64 * 32, h * DH + 64 * N64 + 16 * c, wg * 64, b);
      tma_store_commit();
      tma_store_wait_read<0>();
      mbar_arrive(&empty[buf]);
    }
  }
  if (t == 0) tma_store_wait<0>();
}

template <int DH>
static int launch_attention_short(const void* qkv, void* out, int B, const ShortParams& p, cudaStream_t stream) {
  using L = ShortSmem<DH>;
  CUtensorMap tm[4];
  const uint64_t I = (uint64_t)p.H * DH;
  const uint64_t qdims[3] = {3 * I, (uint64_t)p.N, (uint64_t)B}, qstrides[2] = {6 * I, 6 * I * p.N};
  const uint64_t odims[3] = {I, (uint64_t)p.N, (uint64_t)B}, ostrides[2] = {2 * I, 2 * I * p.N};
  const uint32_t box[3] = {64, SH_KB, 1}, box16[3] = {16, SH_KB, 1};
  int rc = 0;
  if (L::N64) rc = encode_tmap_bf16(&tm[0], qkv, 3, qdims, qstrides, box);
  if (!rc && L::N16) rc = encode_tmap_bf16_sw(&tm[1], qkv, 3, qdims, qstrides, box16, 32);
  if (!rc && L::N64) rc = encode_tmap_bf16(&tm[2], out, 3, odims, ostrides, box);
  if (!rc && L::N16) rc = encode_tmap_bf16_sw(&tm[3], out, 3, odims, ostrides, box16, 0);
  if (rc) return rc;
  // a kind the head does not use gets a copy of the other (never read)
  if (!L::N16) tm[1] = tm[0], tm[3] = tm[2];
  if (!L::N64) tm[0] = tm[1], tm[2] = tm[3];
  auto kern = attention_short_kernel<DH>;
  B200_ENSURE_SMEM(kern, L::BYTES);
  const int grid = p.items < num_sms() ? p.items : num_sms();
  kern<<<grid, SH_THREADS, L::BYTES, stream>>>(tm[0], tm[1], tm[2], tm[3], p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

bool attention_short_ok(int N, int dh) { return N > 128 && N <= SH_ROWS && (dh == 32 || dh == 64); }

int attention_short(const void* qkv, void* out, int B, int N, int H, int dh, float scale_log2e, cudaStream_t stream) {
  ShortParams p{};
  p.N = N;
  p.H = H;
  p.items = B * H;
  p.scale_log2e = scale_log2e;
  return dh == 32 ? launch_attention_short<32>(qkv, out, B, p, stream)
                  : launch_attention_short<64>(qkv, out, B, p, stream);
}

}  // namespace b200
