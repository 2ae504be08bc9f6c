// Kernels of MobileViT (reference mobile_vit.py), for sm_90a.
//   b200vit_attention_groups   softmax attention inside the strided patch groups of B channels-last token maps, heads 8
//                              wide (MobileViTBlock's Transformer(dim, depth, 4, 8, ...), mobile_vit.py:139-159)
//
// The layout follows MaxViT's: token (b, y, x) of a gh x gw map is row (b*gh + y)*gw + x of qkv[B*gh*gw, 3*H*8]
// (packed q | k | v, head-major) and of out[B*gh*gw, H*8].  Group (b, i, j), i < ph, j < pw, is the set of tokens
// (y'*ph + i, x'*pw + j); its token t = y'*(gw/pw) + x' is what rearrange('b d (h ph) (w pw) -> b (ph pw) (h w) d')
// makes of it.  Rows are gathered by that address map; no token is ever copied into group order.
//
// A head 8 wide is too narrow for wgmma (its smallest bf16 K is 16), so the kernel runs mma.sync m16n8k8 for both
// products: S = Q K^T with K = dh = 8 (no padding), and P V per 8 keys with N = dh = 8, each S accumulator tile
// being, as it stands in registers, the A operand of its P tile.  (P V as m16n8k16 would halve its MMAs, but the
// library keeps the 16x8x16 warp-level tensor path out of its SASS; at dh = 8 the exponentials bound the kernel, not
// the MMAs.)  One CTA = one head of `gpc` consecutive groups: it stages their K and V rows (16 B
// each) in shared memory once, zero-filling each group's rows up to `npad`, a whole number of key blocks; its 8 warps
// then take the (group, 16-query slice) items in turn.  A warp loads its slice's Q fragment from global memory and
// streams the group's keys in blocks of KB = 16 NT keys (NT = 4, i.e. 64, unless the whole group is shorter), with an
// fp32 online softmax in log2 units: x = s * (scale log2 e), m the running row max, corr = 2^(m_old - m_new) rescales O
// and the thread's partial l, e = 2^(x - m) (ex2.approx), l sums e in fp32 and P = bf16(e) feeds P V.  At the end l is
// summed over the quad, O * (1 / l) is rounded to bf16 once.  Groups shorter than 16 tokens share a CTA with up to 15
// others, so the CTA does not sit mostly idle.
//
// Bound: at dh = 8 the kernel is limited by the exponential unit: n^2 ex2 per (group, head) against 16 * n dh = 128 n
// bytes of q, k, v and out.
//
// Isolation.  A work item reads only its own group's rows: Q from global memory, K and V from the group's own slice of
// shared memory, whose rows past the group's length are zero (a zero probability times a finite value is 0).  So a
// NaN or Inf stays in its group, and nothing outside the B*gh*gw rows is read or written.  Sums run in a fixed order.
#include "common.cuh"
#include "host_util.h"

namespace {

using namespace b200;

constexpr int GT_THREADS = 256;
constexpr int GT_WARPS = GT_THREADS / 32;

struct GroupParams {
  const __nv_bfloat16* qkv;
  __nv_bfloat16* out;
  int gh, gw, ph, pw;
  int gx;          // gw / pw: tokens per group row
  int n, npad;     // tokens per group; staged rows per group (a multiple of the key block)
  int G, gpc;      // groups in all (B ph pw); groups per CTA
  int nslices;     // 16-query slices per group
  int I;           // H * 8
  float scale_log2e;
};

__device__ __forceinline__ long long group_row(const GroupParams& p, int g, int t) {
  const int b = g / (p.ph * p.pw), ij = g - b * (p.ph * p.pw);
  const int i = ij / p.pw, j = ij - i * p.pw;
  const int yy = t / p.gx, xx = t - yy * p.gx;
  return ((long long)b * p.gh + yy * p.ph + i) * p.gw + xx * p.pw + j;
}

__device__ __forceinline__ void mma_k8(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(b0));
}

__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

__device__ __forceinline__ void ldsm_x2_trans(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

// NT: 16-key chunks per key block (1 to 4; 4 unless the whole group is shorter than 49 tokens)
template <int NT>
__global__ void __launch_bounds__(GT_THREADS)
attention_groups_kernel(const GroupParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int h = blockIdx.y;
  const int g0 = blockIdx.x * p.gpc;
  const int ng = min(p.gpc, p.G - g0);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* sk = smem;                                   // [gpc * npad][16 B]
  uint8_t* sv = smem + (size_t)p.gpc * p.npad * 16;     // [gpc * npad][16 B]
  const uint32_t sk32 = smem_u32(sk), sv32 = smem_u32(sv);

  // stage K and V of the CTA's groups; rows past a group's length are zero
  const int kcol = p.I + h * 8, vcol = 2 * p.I + h * 8;
  const long long ld = 3LL * p.I;
  for (int r = tid; r < ng * p.npad; r += GT_THREADS) {
    const int gl = r / p.npad, t = r - gl * p.npad;
    if (t < p.n) {
      const __nv_bfloat16* src = p.qkv + group_row(p, g0 + gl, t) * ld;
      cp_async16(sk32 + r * 16, src + kcol);
      cp_async16(sv32 + r * 16, src + vcol);
    } else {
      *reinterpret_cast<uint4*>(sk + (size_t)r * 16) = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(sv + (size_t)r * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();

  const int qr = lane >> 2, qc = lane & 3;   // accumulator row (and row + 8), column pair 2 qc
  constexpr int KB = 16 * NT;
  for (int it = warp; it < ng * p.nslices; it += GT_WARPS) {
    const int gl = it / p.nslices, q0 = (it - gl * p.nslices) * 16;
    const int g = g0 + gl;
    // Q fragment (m16n8k8 A): rows q0 + qr and q0 + qr + 8, columns 2 qc, 2 qc + 1; rows past n are zero
    uint32_t qa[2];
    long long orow[2];
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      const int t = q0 + qr + 8 * rh;
      orow[rh] = t < p.n ? group_row(p, g, t) : -1;
      qa[rh] = orow[rh] >= 0 ? *reinterpret_cast<const uint32_t*>(p.qkv + orow[rh] * ld + h * 8 + 2 * qc) : 0u;
    }
    float o[4] = {0.f, 0.f, 0.f, 0.f};
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    // ldmatrix rows: lanes 0-7 the chunk's keys 0-7, lanes 8-15 keys 8-15 (lanes 16-31 repeat them, unused by x2)
    const uint32_t grow = (uint32_t)(gl * p.npad + (lane & 15)) * 16;
    for (int kb = 0; kb < p.npad; kb += KB) {
      float s[2 * NT][4];
#pragma unroll
      for (int c = 0; c < NT; ++c) {
        uint32_t b0, b1;
        ldsm_x2(sk32 + grow + (uint32_t)(kb + 16 * c) * 16, b0, b1);
#pragma unroll
        for (int e = 0; e < 4; ++e) s[2 * c][e] = s[2 * c + 1][e] = 0.f;
        mma_k8(s[2 * c], qa[0], qa[1], b0);
        mma_k8(s[2 * c + 1], qa[0], qa[1], b1);
      }
      // s[tile][e]: row rh = e >> 1, key kb + 8 tile + 2 qc + (e & 1); keys past n get -inf
      const bool tail = kb + KB > p.n;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int tl = 0; tl < 2 * NT; ++tl)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float x = s[tl][e] * p.scale_log2e;
          if (tail && kb + 8 * tl + 2 * qc + (e & 1) >= p.n) x = -INFINITY;
          s[tl][e] = x;
          mx[e >> 1] = fmaxf(mx[e >> 1], x);
        }
      float mu[2];
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 1));
        mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 2));
        const float mn = fmaxf(m[rh], mx[rh]);
        // a row whose scores so far are all -inf subtracts 0: its e are 0, not NaN
        mu[rh] = mn == -INFINITY ? 0.f : mn;
        const float corr = fast_ex2(m[rh] - mu[rh]);
        m[rh] = mn;
        l[rh] *= corr;
        o[2 * rh] *= corr;
        o[2 * rh + 1] *= corr;
      }
#pragma unroll
      for (int c = 0; c < NT; ++c) {
        uint32_t pa[4];
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) {
            const float e0 = fast_ex2(s[2 * c + half][2 * rh] - mu[rh]);
            const float e1 = fast_ex2(s[2 * c + half][2 * rh + 1] - mu[rh]);
            l[rh] += e0 + e1;
            pa[2 * half + rh] = pack_bf16x2(e0, e1);
          }
        uint32_t b0, b1;
        ldsm_x2_trans(sv32 + grow + (uint32_t)(kb + 16 * c) * 16, b0, b1);
        mma_k8(o, pa[0], pa[1], b0);
        mma_k8(o, pa[2], pa[3], b1);
      }
    }
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 1);
      l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 2);
      if (orow[rh] < 0) continue;
      const float inv = 1.0f / l[rh];
      *reinterpret_cast<uint32_t*>(p.out + orow[rh] * p.I + h * 8 + 2 * qc) =
          pack_bf16x2(o[2 * rh] * inv, o[2 * rh + 1] * inv);
    }
  }
}

template <int NT>
int launch_groups(const GroupParams& p, int H, cudaStream_t stream) {
  const size_t smem = 2 * (size_t)p.gpc * p.npad * 16;
  auto kern = attention_groups_kernel<NT>;
  B200_ENSURE_SMEM(kern, smem);
  const dim3 grid((unsigned)((p.G + p.gpc - 1) / p.gpc), (unsigned)H);
  kern<<<grid, GT_THREADS, smem, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace

extern "C" int b200vit_attention_groups(const void* qkv, void* out, int B, int gh, int gw, int ph, int pw, int H,
                                        int dh, float scale, void* stream) {
  B200_CHECK_ARG(qkv && out, "attention_groups: null pointer");
  B200_CHECK_ARG(dh == 8, "attention_groups: dim_head=%d (the kernel is built for 8)", dh);
  B200_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && ph > 0 && pw > 0 && H > 0,
                 "attention_groups: bad shape B=%d map %d x %d groups %d x %d H=%d", B, gh, gw, ph, pw, H);
  B200_CHECK_ARG(gh % ph == 0 && gw % pw == 0, "attention_groups: a %d x %d map is not divisible by %d x %d", gh, gw,
                 ph, pw);
  const long long n = (long long)(gh / ph) * (gw / pw);
  B200_CHECK_ARG(n >= 1 && n <= B200VIT_ATTN_GROUPS_MAX_TOKENS,
                 "attention_groups: %lld tokens per group (1 to %d)", n, B200VIT_ATTN_GROUPS_MAX_TOKENS);
  B200_CHECK_ARG(H <= 65535, "attention_groups: H=%d exceeds the grid", H);
  B200_CHECK_ARG(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
                 "attention_groups: qkv and out must be 16-byte aligned");
  const long long G = (long long)B * ph * pw;
  const int nt = n > 48 ? 4 : (int)((n + 15) / 16);
  GroupParams p{};
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv);
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.gh = gh; p.gw = gw; p.ph = ph; p.pw = pw;
  p.gx = gw / pw;
  p.n = (int)n;
  p.npad = (int)((n + 16 * nt - 1) / (16 * nt) * (16 * nt));
  p.nslices = (int)((n + 15) / 16);
  B200_CHECK_ARG(G <= 0x7fffffffLL, "attention_groups: %lld groups exceed the grid", G);
  // two items per warp where the groups are short: short groups share a CTA
  long long per = 2 * GT_WARPS / p.nslices;
  per = per < 1 ? 1 : (per > G ? G : per);
  p.gpc = (int)per;
  p.G = (int)G;
  p.I = H * 8;
  p.scale_log2e = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (nt) {
    case 1: return launch_groups<1>(p, H, st);
    case 2: return launch_groups<2>(p, H, st);
    case 3: return launch_groups<3>(p, H, st);
    default: return launch_groups<4>(p, H, st);
  }
}
