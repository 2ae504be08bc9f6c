// HBM-bound row kernels around the GEMMs: LayerNorm, patchify + LayerNorm, token assembly, mean pool, cast.
// One warp per row, float4 / 16-byte accesses, fp32 statistics (two-pass variance, eps inside the sqrt -- the
// semantics of torch.nn.LayerNorm used at vit.py:19,39,69,101,103).  The token rows that leave embed_tokens,
// embed_varlen and rowstats_cast with LN-fold statistics are all written through emit_row_stats (common.cuh).
#include "common.cuh"
#include "host_util.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm: x fp32 [*, D] -> bf16 and/or fp32 (row statistics: ln_row_stats, common.cuh)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ gamma,
                 const float* __restrict__ beta, __nv_bfloat16* __restrict__ out_bf16, float* __restrict__ out_f32,
                 long long ldo, const int* __restrict__ row_index, int M, int D, float eps) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const long long src = row_index ? (long long)row_index[row] : (long long)row;
  const float* xr = x + src * ldx;
  float mean, rstd;
  ln_row_stats(xr, D, lane, mean, rstd, eps);
  const bool vec = ((D & 3) == 0) && ((ldo & 3) == 0);
  if (vec) {
    for (int i = lane * 4; i < D; i += 128) {
      const float4 v = *reinterpret_cast<const float4*>(xr + i);
      const float4 g = *reinterpret_cast<const float4*>(gamma + i);
      float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
      if (beta) b = *reinterpret_cast<const float4*>(beta + i);
      float4 y;
      y.x = (v.x - mean) * rstd * g.x + b.x;
      y.y = (v.y - mean) * rstd * g.y + b.y;
      y.z = (v.z - mean) * rstd * g.z + b.z;
      y.w = (v.w - mean) * rstd * g.w + b.w;
      if (out_f32) *reinterpret_cast<float4*>(out_f32 + (long long)row * ldo + i) = y;
      if (out_bf16) {
        uint2 pk;
        pk.x = pack_bf16x2(y.x, y.y);
        pk.y = pack_bf16x2(y.z, y.w);
        *reinterpret_cast<uint2*>(out_bf16 + (long long)row * ldo + i) = pk;
      }
    }
  } else {
    for (int i = lane; i < D; i += 32) {
      const float y = (xr[i] - mean) * rstd * gamma[i] + (beta ? beta[i] : 0.f);
      if (out_f32) out_f32[(long long)row * ldo + i] = y;
      if (out_bf16) out_bf16[(long long)row * ldo + i] = __float2bfloat16_rn(y);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Patchify + LayerNorm(patch_dim).  One CTA per (image, patch row): the C x ph x W pixel slab is staged in smem with
// coalesced 16-byte loads, then each warp normalises whole patches and writes bf16 rows in (p1 p2 c) order.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
patchify_ln_kernel(const __nv_bfloat16* __restrict__ img, const float* __restrict__ gamma,
                   const float* __restrict__ beta, __nv_bfloat16* __restrict__ out, long long ldo, int nrows, int C,
                   int H, int W, int ph, int pw, float eps) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* slab = reinterpret_cast<__nv_bfloat16*>(smem_raw);  // [C][ph][W]
  const int gh = H / ph, gw = W / pw;
  const int slab_elems = C * ph * W;
  const int row_elems = ph * W;  // contiguous per channel in global memory
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pd = ph * pw * C;
  // Output element e = (p1*pw + p2)*C + c lives at slab[(c*ph + p1)*W + w*pw + p2].  Each lane owns the element PAIRS
  // e = 2*lane + 64*k (so it stores 4 bytes at a time, 128 B per warp); the slab offsets of its pairs do not depend on
  // the patch (b, h, w), so they are computed once per (persistent) CTA and kept in registers with gamma / beta.
  constexpr int MAXP = 12;  // pairs per lane held in registers: covers patch_dim <= 768 (16x16x3)
  const int npairs = (pd + 1) / 2;
  int off0[MAXP], off1[MAXP];
  float g0[MAXP], g1[MAXP], b0[MAXP], b1[MAXP];
  const bool fast = npairs <= 32 * MAXP && (pd & 1) == 0;
  if (fast) {
#pragma unroll
    for (int k = 0; k < MAXP; ++k) {
      const int e = 2 * (lane + 32 * k);
      off0[k] = off1[k] = -1;
      g0[k] = g1[k] = b0[k] = b1[k] = 0.f;
      if (e < pd) {
        int c = e % C, pp = e / C;
        off0[k] = (c * ph + pp / pw) * W + pp % pw;
        g0[k] = gamma[e];
        b0[k] = beta[e];
        c = (e + 1) % C;
        pp = (e + 1) / C;
        off1[k] = (c * ph + pp / pw) * W + pp % pw;
        g1[k] = gamma[e + 1];
        b1[k] = beta[e + 1];
      }
    }
  }
  for (int bh = blockIdx.x; bh < nrows; bh += gridDim.x) {
  const int b = bh / gh, h = bh % gh;
  __syncthreads();  // previous slab fully consumed
  if ((row_elems & 7) == 0 && ((H * W) & 7) == 0) {
    for (int i = threadIdx.x * 8; i < slab_elems; i += blockDim.x * 8) {
      const int c = i / row_elems, r = i % row_elems;
      const __nv_bfloat16* src = img + ((long long)(b * C + c) * H + (long long)h * ph) * W + r;
      *reinterpret_cast<uint4*>(slab + i) = *reinterpret_cast<const uint4*>(src);
    }
  } else {
    for (int i = threadIdx.x; i < slab_elems; i += blockDim.x) {
      const int c = i / row_elems, r = i % row_elems;
      slab[i] = img[((long long)(b * C + c) * H + (long long)h * ph) * W + r];
    }
  }
  __syncthreads();
  for (int w = warp; w < gw; w += 8) {
    __nv_bfloat16* orow = out + ((long long)(b * gh + h) * gw + w) * ldo;
    if (fast) {
      const __nv_bfloat16* sl = slab + w * pw;
      float v0[MAXP], v1[MAXP];
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < MAXP; ++k) {
        v0[k] = off0[k] >= 0 ? __bfloat162float(sl[off0[k]]) : 0.f;
        v1[k] = off1[k] >= 0 ? __bfloat162float(sl[off1[k]]) : 0.f;
        s += v0[k] + v1[k];
      }
      const float mean = warp_sum(s) / (float)pd;
      float q = 0.f;
#pragma unroll
      for (int k = 0; k < MAXP; ++k) {
        const float d0 = off0[k] >= 0 ? v0[k] - mean : 0.f;
        const float d1 = off1[k] >= 0 ? v1[k] - mean : 0.f;
        q = fmaf(d0, d0, fmaf(d1, d1, q));
      }
      const float rstd = rsqrtf(warp_sum(q) / (float)pd + eps);
#pragma unroll
      for (int k = 0; k < MAXP; ++k) {
        const int e = 2 * (lane + 32 * k);
        if (e < (int)ldo) {
          uint32_t pk = 0u;  // columns [pd, ldo) are zero (K padding)
          if (off0[k] >= 0)
            pk = pack_bf16x2((v0[k] - mean) * rstd * g0[k] + b0[k], (v1[k] - mean) * rstd * g1[k] + b1[k]);
          *reinterpret_cast<uint32_t*>(orow + e) = pk;
        }
      }
      for (int e = 2 * 32 * MAXP + lane; e < (int)ldo; e += 32) orow[e] = __float2bfloat16_rn(0.f);
      continue;
    }
    // generic path (odd patch_dim or very large patches)
    float s = 0.f;
    for (int e = lane; e < pd; e += 32) {
      const int c = e % C, pp = e / C, p2 = pp % pw, p1 = pp / pw;
      s += __bfloat162float(slab[(c * ph + p1) * W + w * pw + p2]);
    }
    const float mean = warp_sum(s) / (float)pd;
    float q = 0.f;
    for (int e = lane; e < pd; e += 32) {
      const int c = e % C, pp = e / C, p2 = pp % pw, p1 = pp / pw;
      const float d = __bfloat162float(slab[(c * ph + p1) * W + w * pw + p2]) - mean;
      q += d * d;
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)pd + eps);
    for (int e = lane; e < (int)ldo; e += 32) {
      float y = 0.f;
      if (e < pd) {
        const int c = e % C, pp = e / C, p2 = pp % pw, p1 = pp / pw;
        y = (__bfloat162float(slab[(c * ph + p1) * W + w * pw + p2]) - mean) * rstd * gamma[e] + beta[e];
      }
      orow[e] = __float2bfloat16_rn(y);
    }
  }
  }  // persistent loop over (image, patch row)
}

// 16 x 16 patches, 3 channels, 16-byte aligned rows (W % 8 == 0): the ViT-B/L geometry.  Slab rows are padded so that
// the 16-byte chunk reads of a patch are bank-conflict free (row stride = 16 bytes mod 64); lane (p1, half) reads 8
// pixels of each channel, interleaves them to the 24 consecutive (p1 p2 c) outputs it owns and writes three 16-byte
// pieces -- every patch is read from shared memory once with 128-bit loads and leaves as coalesced 48-byte runs.
// gamma / beta are staged in shared memory once per (persistent) CTA.
__global__ void __launch_bounds__(256)
patchify_ln16c3_kernel(const __nv_bfloat16* __restrict__ img, const float* __restrict__ gamma,
                       const float* __restrict__ beta, __nv_bfloat16* __restrict__ out, long long ldo, int nrows,
                       int H, int W, int wp, float eps) {
  constexpr int C = 3, P = 16, PD = C * P * P;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float* sg = reinterpret_cast<float*>(smem_raw);         // [768] gamma
  float* sb = sg + PD;                                    // [768] beta
  __nv_bfloat16* slab = reinterpret_cast<__nv_bfloat16*>(sb + PD);  // [C*16][wp]
  const int gh = H / P, gw = W / P;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < PD; i += blockDim.x) {
    sg[i] = gamma[i];
    sb[i] = beta[i];
  }
  const int vpr = W >> 3;
  const int p1 = lane >> 1, half = lane & 1;
  const int e0 = (p1 * P + half * 8) * C;  // first of this lane's 24 output elements
  for (int bh = blockIdx.x; bh < nrows; bh += gridDim.x) {
    const int b = bh / gh, h = bh % gh;
    __syncthreads();  // previous slab fully consumed (and gamma / beta staged)
    for (int i = threadIdx.x; i < C * P * vpr; i += blockDim.x) {
      const int rowi = i / vpr, vx = i - rowi * vpr;
      const int c = rowi >> 4, r = rowi & 15;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(img + ((long long)(b * C + c) * H + h * P + r) * W) + vx);
      *(reinterpret_cast<uint4*>(slab + (long long)rowi * wp) + vx) = v;
    }
    __syncthreads();
    for (int w = warp; w < gw; w += 8) {
      float f[C][8];
      float sum = 0.f;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const uint4 raw = *reinterpret_cast<const uint4*>(slab + (long long)(c * P + p1) * wp + w * P + half * 8);
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 t = __bfloat1622float2(h2[i]);
          f[c][2 * i] = t.x;
          f[c][2 * i + 1] = t.y;
          sum += t.x + t.y;
        }
      }
      const float mean = warp_sum(sum) * (1.0f / PD);
      float q = 0.f;
#pragma unroll
      for (int c = 0; c < C; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[c][i] - mean;
          q = fmaf(d, d, q);
        }
      const float rstd = rsqrtf(warp_sum(q) * (1.0f / PD) + eps);
      __nv_bfloat16* orow = out + ((long long)(b * gh + h) * gw + w) * ldo;
      // outputs e0 + j, j = px*3 + c, in three groups of 8
      float y[24];
#pragma unroll
      for (int px = 0; px < 8; ++px)
#pragma unroll
        for (int c = 0; c < C; ++c) {
          const int j = px * C + c;
          y[j] = (f[c][px] - mean) * rstd * sg[e0 + j] + sb[e0 + j];
        }
#pragma unroll
      for (int g = 0; g < 3; ++g) {
        uint4 pk;
        pk.x = pack_bf16x2(y[8 * g], y[8 * g + 1]);
        pk.y = pack_bf16x2(y[8 * g + 2], y[8 * g + 3]);
        pk.z = pack_bf16x2(y[8 * g + 4], y[8 * g + 5]);
        pk.w = pack_bf16x2(y[8 * g + 6], y[8 * g + 7]);
        *reinterpret_cast<uint4*>(orow + e0 + 8 * g) = pk;
      }
      for (int e = PD + lane; e < (int)ldo; e += 32) orow[e] = __float2bfloat16_rn(0.f);  // K padding
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Shifted patch tokenization + LayerNorm(5 C p^2) (SPT, vit_for_small_dataset.py:81-96).  One CTA per (image, patch
// row), persistent: the p + 2 image rows the patch row and its vertical shifts read are staged per channel in shared
// memory, SPT_LPAD columns right of a zero column for x = -1 and with one zero column at x = W, the rows above / below
// the image zero -- so each of the five sources is a fixed offset into the slab and needs no bounds test.  A table of
// those offsets per output column (patch-relative, built once per CTA) replaces the (p1 p2 k c) index arithmetic; each
// warp normalises whole patches (two passes over the slab for mean and variance, one to write) in 16-byte pieces.
// ---------------------------------------------------------------------------------------------------------------
constexpr int SPT_LPAD = 8;  // slab column of x = 0 (keeps the staged rows 16-byte aligned); x = -1 is column 7

__global__ void __launch_bounds__(256)
patchify_spt_ln_kernel(const __nv_bfloat16* __restrict__ img, const float* __restrict__ gamma,
                       const float* __restrict__ beta, __nv_bfloat16* __restrict__ out, long long ldo, int nrows, int C,
                       int H, int W, int p, int rs, float eps) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int pd = 5 * C * p * p, C5 = 5 * C, ps = p + 2;
  int* offs = reinterpret_cast<int*>(smem_raw);                                  // [pd rounded up to 8]
  __nv_bfloat16* slab = reinterpret_cast<__nv_bfloat16*>(offs + ((pd + 7) & ~7));  // [C][p + 2][rs]
  const int gh = H / p, gw = W / p;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int e = threadIdx.x; e < pd; e += blockDim.x) {
    const int pix = e / C5, kc = e - pix * C5, k = kc / C, c = kc - k * C;
    const int p1 = pix / p, p2 = pix - p1 * p;
    const int dx = k == 1 ? -1 : k == 2 ? 1 : 0, dy = k == 3 ? -1 : k == 4 ? 1 : 0;
    offs[e] = (c * ps + 1 + p1 + dy) * rs + SPT_LPAD + p2 + dx;
  }
  const int slab_rows = C * ps;
  for (int r = threadIdx.x; r < slab_rows; r += blockDim.x) {  // the x = -1 and x = W columns stay zero
    slab[r * rs + SPT_LPAD - 1] = __float2bfloat16_rn(0.f);
    slab[r * rs + SPT_LPAD + W] = __float2bfloat16_rn(0.f);
  }
  const bool vec = (W & 7) == 0 && (reinterpret_cast<uintptr_t>(img) & 15) == 0;
  const int vpr = vec ? W >> 3 : W;  // work items per slab row
  const int nchunks = (int)(ldo >> 3);
  for (int bh = blockIdx.x; bh < nrows; bh += gridDim.x) {
    const int b = bh / gh, h = bh % gh;
    __syncthreads();  // previous slab fully consumed (and the table / pad columns written)
    for (int i = threadIdx.x; i < slab_rows * vpr; i += blockDim.x) {
      const int r = i / vpr, v = i - r * vpr;
      const int c = r / ps, y = h * p - 1 + (r - c * ps);
      const bool in = y >= 0 && y < H;
      const __nv_bfloat16* src = img + ((long long)(b * C + c) * H + y) * W;
      __nv_bfloat16* dst = slab + r * rs + SPT_LPAD;
      if (vec) {
        const uint4 u = in ? __ldg(reinterpret_cast<const uint4*>(src) + v) : make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(dst + 8 * v) = u;
      } else {
        dst[v] = in ? src[v] : __float2bfloat16_rn(0.f);
      }
    }
    __syncthreads();
    for (int w = warp; w < gw; w += 8) {
      const __nv_bfloat16* sl = slab + w * p;
      float s = 0.f;
      for (int e = lane; e < pd; e += 32) s += __bfloat162float(sl[offs[e]]);
      const float mean = warp_sum(s) / (float)pd;
      float q = 0.f;
      for (int e = lane; e < pd; e += 32) {
        const float d = __bfloat162float(sl[offs[e]]) - mean;
        q = fmaf(d, d, q);
      }
      const float rstd = rsqrtf(warp_sum(q) / (float)pd + eps);
      __nv_bfloat16* orow = out + ((long long)(b * gh + h) * gw + w) * ldo;
      for (int ch = lane; ch < nchunks; ch += 32) {
        const int e0 = ch * 8;
        float y[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int e = e0 + j;  // columns [pd, ldo) are zero (K padding)
          y[j] = e < pd ? (__bfloat162float(sl[offs[e]]) - mean) * rstd * __ldg(gamma + e) + __ldg(beta + e) : 0.f;
        }
        uint4 pk;
        pk.x = pack_bf16x2(y[0], y[1]);
        pk.y = pack_bf16x2(y[2], y[3]);
        pk.z = pack_bf16x2(y[4], y[5]);
        pk.w = pack_bf16x2(y[6], y[7]);
        *reinterpret_cast<uint4*>(orow + e0) = pk;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Token assembly: LN(dim) of the patch projection + positional embedding + cls row  -> fp32 residual stream
// ---------------------------------------------------------------------------------------------------------------
// POS = false: no positional term (vit_nd_rotary.py:272-287 has no table; rotary positions act on q / k instead)
// LN = false: no LayerNorm(dim), the patch rows are y itself (SPT, vit_for_small_dataset.py:127-132)
template <bool POS, bool LN>
__global__ void __launch_bounds__(256)
embed_tokens_kernel(const float* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                    const float* __restrict__ cls, const float* __restrict__ pos, float* __restrict__ x,
                    __nv_bfloat16* __restrict__ xb, float* __restrict__ stats, int B, int n, int ncls, int D,
                    float eps, const float* __restrict__ tail, int ntail, int pos_period, int pos_stride,
                    int cls_pos) {
  const int N = n + ncls + ntail;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= (long long)B * N) return;
  const int b = (int)(row / N), t = (int)(row % N);
  float* xr = x + row * D;
  __nv_bfloat16* xbr = xb ? xb + row * D : nullptr;
  // positional row: group b reads the table block (b % pos_period) * pos_stride; the cls rows take the first rows of
  // the block when cls_pos, else no position (vivit.py:227-231); tail rows carry no positional embedding
  const int tc = min(t, n + ncls - 1);
  const long long prow = (long long)(b % pos_period) * pos_stride + (cls_pos ? tc : max(tc - ncls, 0));
  const float* pr = POS ? pos + prow * D : nullptr;
  // every row kind goes through emit_row_stats: the first layer's LN-fold statistics are the bits rowstats_cast
  // would write for the same fp32 row
  float* st = stats ? stats + 2 * row : nullptr;
  auto ld4 = [](const float* p) { return *reinterpret_cast<const float4*>(p); };
  auto add4 = [](float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); };
  if (t < ncls) {
    const float* cr = cls + (long long)t * D;
    if (POS && cls_pos)
      emit_row_stats<true>(D, lane, xr, xbr, st, [&](int i) { return add4(ld4(cr + i), ld4(pr + i)); },
                     [&](int i) { return cr[i] + pr[i]; });
    else
      emit_row_stats<true>(D, lane, xr, xbr, st, [&](int i) { return ld4(cr + i); }, [&](int i) { return cr[i]; });
  } else if (t >= ncls + n) {  // register tokens appended after the patches (simple_vit_with_register_tokens.py:124-126)
    const float* tr = tail + (long long)(t - ncls - n) * D;
    emit_row_stats<true>(D, lane, xr, xbr, st, [&](int i) { return ld4(tr + i); }, [&](int i) { return tr[i]; });
  } else if (!LN) {
    const float* yr = y + ((long long)b * n + (t - ncls)) * D;
    if (POS)
      emit_row_stats<true>(D, lane, xr, xbr, st, [&](int i) { return add4(ld4(yr + i), ld4(pr + i)); },
                     [&](int i) { return yr[i] + pr[i]; });
    else
      emit_row_stats<true>(D, lane, xr, xbr, st, [&](int i) { return ld4(yr + i); }, [&](int i) { return yr[i]; });
  } else {
    const float* yr = y + ((long long)b * n + (t - ncls)) * D;
    float mean, rstd;
    ln_row_stats(yr, D, lane, mean, rstd, eps);
    // ((LN . gamma + beta) + pos): the association of the reference's x + pos_embedding
    auto ln1 = [&](int i) {
      const float v = (yr[i] - mean) * rstd * gamma[i] + beta[i];
      return POS ? v + pr[i] : v;
    };
    auto ln4 = [&](int i) {
      const float4 v = ld4(yr + i), g = ld4(gamma + i), be = ld4(beta + i);
      float4 o;
      o.x = (v.x - mean) * rstd * g.x + be.x;
      o.y = (v.y - mean) * rstd * g.y + be.y;
      o.z = (v.z - mean) * rstd * g.z + be.z;
      o.w = (v.w - mean) * rstd * g.w + be.w;
      return POS ? add4(o, ld4(pr + i)) : o;
    };
    emit_row_stats<true>(D, lane, xr, xbr, st, ln4, ln1);
  }
}

// fp32 rows -> bf16 copy + (sum, sum of squares) of the bf16-rounded row: entry into the LN-folded layer chain for
// token matrices that do not come from embed_tokens (Transformer called directly on tokens).
__global__ void __launch_bounds__(256)
rowstats_cast_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ xb, float* __restrict__ stats, int M,
                     int D) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  rowstats_cast_row(x + row * D, xb + row * D, stats + 2 * row, D, lane);
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
mean_pool_kernel(const float* __restrict__ x, float* __restrict__ out, int N, int D, int n_pool) {
  const int b = blockIdx.y;
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  const float* xp = x + (long long)b * N * D + d;
  float s = 0.f;
  for (int t = 0; t < n_pool; ++t) s += xp[(long long)t * D];
  out[(long long)b * D + d] = s / (float)n_pool;
}

__global__ void __launch_bounds__(256)
cast_f32_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, long long n) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const float4 a = *reinterpret_cast<const float4*>(x + i);
    const float4 b = *reinterpret_cast<const float4*>(x + i + 4);
    uint4 pk;
    pk.x = pack_bf16x2(a.x, a.y);
    pk.y = pack_bf16x2(a.z, a.w);
    pk.z = pack_bf16x2(b.x, b.y);
    pk.w = pack_bf16x2(b.z, b.w);
    *reinterpret_cast<uint4*>(out + i) = pk;
  } else {
    for (long long j = i; j < n; ++j) out[j] = __float2bfloat16_rn(x[j]);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200vit_layernorm(const float* x, int64_t ldx, const float* gamma, const float* beta, void* out_bf16,
                                 float* out_f32, int64_t ldo, const int32_t* row_index, int M, int D, float eps,
                                 void* stream) {
  B200_CHECK_ARG(x && gamma && (out_bf16 || out_f32), "layernorm: null pointer");
  B200_CHECK_ARG(M > 0 && D > 0 && ldx >= D && ldo >= D, "layernorm: bad shape M=%d D=%d", M, D);
  B200_CHECK_ARG((ldx & 3) == 0 || (D & 3) != 0, "layernorm: ldx must be a multiple of 4 when D is");
  layernorm_kernel<<<(M + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, ldx, gamma, beta, reinterpret_cast<__nv_bfloat16*>(out_bf16), out_f32, ldo, row_index, M, D, eps);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_patchify_ln(const void* img, const float* gamma, const float* beta, void* out_bf16, int64_t ldo,
                                   int B, int C, int H, int W, int ph, int pw, float eps, void* stream) {
  B200_CHECK_ARG(img && gamma && beta && out_bf16, "patchify_ln: null pointer");
  B200_CHECK_ARG(B > 0 && C > 0 && ph > 0 && pw > 0 && H % ph == 0 && W % pw == 0,
                 "patchify_ln: image %dx%d not divisible by patch %dx%d", H, W, ph, pw);
  B200_CHECK_ARG(ldo >= (int64_t)C * ph * pw, "patchify_ln: ldo too small");
  const bool fast = C == 3 && ph == 16 && pw == 16 && (W % 8) == 0 && ((long long)H * W) % 8 == 0 && (ldo % 8) == 0 &&
                    (reinterpret_cast<uintptr_t>(img) & 15) == 0 && (reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0;
  const int wp = (W + 31) / 32 * 32 + 16;  // fast path: padded slab row (stride = 16 bytes mod 64: no bank conflicts)
  const size_t smem = fast ? (size_t)C * 16 * wp * 2 + 2 * 768 * sizeof(float) : (size_t)C * ph * W * 2;
  B200_CHECK_ARG(smem <= 200 * 1024, "patchify_ln: patch-row slab of %zu bytes exceeds shared memory", smem);
  if (fast) B200_ENSURE_SMEM(patchify_ln16c3_kernel, smem);
  else B200_ENSURE_SMEM(patchify_ln_kernel, smem);
  const int nrows = B * (H / ph);
  const int per_sm = (int)(200 * 1024 / (smem + 1024)) < 8 ? (int)(200 * 1024 / (smem + 1024)) : 8;
  int grid = num_sms() * (per_sm < 1 ? 1 : per_sm);
  if (grid > nrows) grid = nrows;
  auto st = reinterpret_cast<cudaStream_t>(stream);
  if (fast)
    patchify_ln16c3_kernel<<<grid, 256, smem, st>>>(reinterpret_cast<const __nv_bfloat16*>(img), gamma, beta,
                                                    reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, nrows, H, W, wp,
                                                    eps);
  else
    patchify_ln_kernel<<<grid, 256, smem, st>>>(reinterpret_cast<const __nv_bfloat16*>(img), gamma, beta,
                                                reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, nrows, C, H, W, ph, pw,
                                                eps);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_patchify_spt_ln(const void* img, const float* gamma, const float* beta, void* out_bf16,
                                       int64_t ldo, int B, int C, int H, int W, int p, float eps, void* stream) {
  B200_CHECK_ARG(img && gamma && beta && out_bf16, "patchify_spt_ln: null pointer");
  B200_CHECK_ARG(B > 0 && C > 0 && p > 0 && H > 0 && W > 0 && H % p == 0 && W % p == 0,
                 "patchify_spt_ln: image %dx%d not divisible by patch %d", H, W, p);
  const long long pd = 5LL * C * p * p;
  B200_CHECK_ARG(ldo >= pd && ldo % 8 == 0, "patchify_spt_ln: ldo=%lld must be >= 5*C*p*p=%lld and a multiple of 8",
                 (long long)ldo, pd);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0, "patchify_spt_ln: out must be 16-byte aligned");
  const int rs = (W + SPT_LPAD + 1 + 7) / 8 * 8;  // slab row: zero column, W pixels, zero column, 16-byte multiple
  const size_t smem = (size_t)((pd + 7) & ~7LL) * sizeof(int) + (size_t)C * (p + 2) * rs * 2;
  B200_CHECK_ARG(smem <= 200 * 1024, "patchify_spt_ln: patch-row slab of %zu bytes exceeds shared memory", smem);
  B200_ENSURE_SMEM(patchify_spt_ln_kernel, smem);
  const int nrows = B * (H / p);
  const int per_sm = (int)(200 * 1024 / (smem + 1024)) < 8 ? (int)(200 * 1024 / (smem + 1024)) : 8;
  int grid = num_sms() * (per_sm < 1 ? 1 : per_sm);
  if (grid > nrows) grid = nrows;
  patchify_spt_ln_kernel<<<grid, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(img), gamma, beta, reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, nrows,
      C, H, W, p, rs, eps);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_rowstats_cast(const float* x, void* xb_bf16, float* stats, int M, int D, void* stream) {
  B200_CHECK_ARG(x && xb_bf16 && stats && M > 0 && D > 0, "rowstats_cast: bad argument");
  rowstats_cast_kernel<<<(M + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, reinterpret_cast<__nv_bfloat16*>(xb_bf16), stats, M, D);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_embed_tokens_grouped(const float* y, const float* gamma, const float* beta, const float* cls,
                                            const float* pos, const float* tail, float* x, void* xb_bf16, float* stats,
                                            int groups, int n, int ncls, int ntail, int D, float eps, int pos_period,
                                            int pos_stride, int cls_pos, void* stream) {
  B200_CHECK_ARG(y && (beta || !gamma) && x, "embed_tokens: null pointer");
  B200_CHECK_ARG(ncls == 0 || cls, "embed_tokens: ncls=%d without cls", ncls);
  B200_CHECK_ARG(ntail == 0 || tail, "embed_tokens: ntail=%d without tail", ntail);
  B200_CHECK_ARG(groups > 0 && n > 0 && D > 0 && ncls >= 0 && ntail >= 0, "embed_tokens: bad shape");
  B200_CHECK_ARG(pos_period > 0 && pos_stride >= 0, "embed_tokens: bad positional period %d / stride %d", pos_period,
                 pos_stride);
  const long long rows = (long long)groups * (n + ncls + ntail);
  auto kern = gamma ? (pos ? embed_tokens_kernel<true, true> : embed_tokens_kernel<false, true>)
                    : (pos ? embed_tokens_kernel<true, false> : embed_tokens_kernel<false, false>);
  kern<<<(unsigned)((rows + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      y, gamma, beta, cls, pos, x, reinterpret_cast<__nv_bfloat16*>(xb_bf16), stats, groups, n, ncls, D, eps, tail,
      ntail, pos_period, pos_stride, cls_pos != 0);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_embed_tokens(const float* y, const float* gamma, const float* beta, const float* cls,
                                    const float* pos, const float* tail, float* x, void* xb_bf16, float* stats, int B,
                                    int n, int ncls, int ntail, int D, float eps, void* stream) {
  // one table for every image, the cls rows positioned first
  return b200vit_embed_tokens_grouped(y, gamma, beta, cls, pos, tail, x, xb_bf16, stats, B, n, ncls, ntail, D, eps, 1,
                                      0, 1, stream);
}

extern "C" int b200vit_mean_pool(const float* x, float* out, int B, int N, int D, int n_pool, void* stream) {
  B200_CHECK_ARG(x && out && B > 0 && N > 0 && D > 0, "mean_pool: bad argument");
  B200_CHECK_ARG(n_pool > 0 && n_pool <= N, "mean_pool: n_pool=%d outside (0, N=%d]", n_pool, N);
  dim3 grid((D + 255) / 256, B);
  mean_pool_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, out, N, D, n_pool);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_cast_f32_bf16(const float* x, void* out_bf16, int64_t n, void* stream) {
  B200_CHECK_ARG(x && out_bf16 && n > 0, "cast: bad argument");
  const long long blocks = (n / 8 + 255) / 256 + 1;
  cast_f32_bf16_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, reinterpret_cast<__nv_bfloat16*>(out_bf16), n);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// NaViT: per-head q/k RMSNorm on the packed qkv buffer, in place (reference na_vit.py:93-101,149-150):
//   v <- v / max(||v||_2, 1e-12) * sqrt(dh) * gamma[h, d]      for the q and k slices of every token and head.
// gamma_qk: fp32 [2][H][dh] (q first), sqrt(dh) NOT folded in.  One warp per token, 16 bytes per lane and step.
// ---------------------------------------------------------------------------------------------------------------
namespace b200 {

template <int DH>
struct HeadLanes {
  static constexpr int CH = DH / 8;                                    // 16-byte chunks per head
  static constexpr int LPH = CH <= 4 ? 4 : CH <= 8 ? 8 : 16;            // lanes per head: CH rounded up to a power of 2
  static constexpr int HPS = 32 / LPH;                                 // heads per warp and step
  static constexpr float SQRT_DH = DH == 32 ? 5.656854249492380f : DH == 64 ? 8.0f : DH == 80 ? 8.944271909999159f
                                                                                            : 11.313708498984761f;
  static_assert(CH * 8 == DH && CH <= 16, "head width");
};

// buf[T, ld] bf16: the `nheads` consecutive DH-wide heads starting at the row's column 0 are normalised in place.
// One warp per token; LPH lanes per head (8 bf16 = 16 B each; dh 80 = 10 chunks leaves 6 of its 16 lanes idle, their
// zeros join the sums of the values), so HPS heads are normalised per step with a butterfly inside each LPH-lane
// group; the loads of U steps are issued before the first reduction (a serial load -> shuffle -> store chain per step
// left the kernel latency bound at a quarter of the HBM rate).  Each lane's part of a sum is a chain of 8 fp32 adds or
// fmas, then log2(LPH) butterfly levels.
// LN = true: LayerNorm over the head's DH values without bias, (v - mean) * rsqrt(var + eps) * gamma with a two-pass
// variance (the idle lanes of dh 80 masked out of the second pass) -- the q / k norm of the nested-tensor NaViT
// (na_vit_nested_tensor.py:61-62,101-102) -- instead of the RMS norm.
template <int DH, int U, bool LN>
__global__ void __launch_bounds__(256)
rmsnorm_heads_kernel(__nv_bfloat16* __restrict__ buf, long long ld, const float* __restrict__ gamma, int T,
                     int nheads, float eps) {
  using HL = HeadLanes<DH>;
  constexpr int LPH = HL::LPH, HPS = HL::HPS;
  const long long t = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  __nv_bfloat16* row = buf + t * ld;
  const int sub = lane % LPH, grp = lane / LPH;
  const bool act = sub < HL::CH;  // (always true unless dh = 80)
  for (int base = 0; base < nheads; base += HPS * U) {
    uint4 raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int hh = base + HPS * u + grp;  // (heads beyond nheads: the group only joins the shuffles)
      raw[u] = act ? *(reinterpret_cast<const uint4*>(row + (hh < nheads ? hh : 0) * DH) + sub)
                   : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int hh = base + HPS * u + grp;
      __nv_bfloat162* h2 = reinterpret_cast<__nv_bfloat162*>(&raw[u]);
      float2 f[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) f[i] = __bfloat1622float2(h2[i]);
      float inv;
      if (LN) {
        // two-pass variance over the values held in registers: E[x^2] - mean^2 loses var to cancellation in fp32 once
        // |mean| / std reaches the hundreds
        float s1 = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) s1 += f[i].x + f[i].y;
#pragma unroll
        for (int o = LPH / 2; o > 0; o >>= 1) s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        const float mean = s1 * (1.0f / (float)DH);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          f[i].x -= mean;
          f[i].y -= mean;
          q = fmaf(f[i].x, f[i].x, fmaf(f[i].y, f[i].y, q));
        }
        if (!act) q = 0.f;  // dh 80: an idle lane's zeros would add (0 - mean)^2
#pragma unroll
        for (int o = LPH / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
        inv = rsqrtf(q * (1.0f / (float)DH) + eps);
      } else {
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) ss = fmaf(f[i].x, f[i].x, fmaf(f[i].y, f[i].y, ss));
#pragma unroll
        for (int o = LPH / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        // max(||v||, 1e-12) as torch's clamp_min: a NaN norm stays NaN (fmaxf would return 1e-12 and turn the head's
        // other values into finite garbage)
        const float nrm = sqrtf(ss);
        inv = HL::SQRT_DH / (nrm < 1e-12f ? 1e-12f : nrm);
      }
      if (hh < nheads && act) {
        const float4 g0 = *reinterpret_cast<const float4*>(gamma + hh * DH + 8 * sub);
        const float4 g1 = *reinterpret_cast<const float4*>(gamma + hh * DH + 8 * sub + 4);
        h2[0] = __floats2bfloat162_rn(f[0].x * inv * g0.x, f[0].y * inv * g0.y);
        h2[1] = __floats2bfloat162_rn(f[1].x * inv * g0.z, f[1].y * inv * g0.w);
        h2[2] = __floats2bfloat162_rn(f[2].x * inv * g1.x, f[2].y * inv * g1.y);
        h2[3] = __floats2bfloat162_rn(f[3].x * inv * g1.z, f[3].y * inv * g1.w);
        *(reinterpret_cast<uint4*>(row + hh * DH) + sub) = raw[u];
      }
    }
  }
}

// SepViT's window-token pre-norm and activation (reference sep_vit.py:96-98), in place on buf[T, ld] bf16:
//   v <- GELU_erf((v - mean) * rsqrt(var + eps) * gamma[d] + beta[d])  over each of the `nheads` DH-wide heads, one
// nn.LayerNorm(dh) shared by the heads.  The lane layout, the sums and the two-pass variance are those of
// rmsnorm_heads_kernel<DH, 1, true>; GELU is common.cuh's gelu_erf, as the GEMM epilogue's.
template <int DH>
__global__ void __launch_bounds__(256)
head_layernorm_gelu_kernel(__nv_bfloat16* __restrict__ buf, long long ld, const float* __restrict__ gamma,
                           const float* __restrict__ beta, int T, int nheads, float eps) {
  using HL = HeadLanes<DH>;
  constexpr int LPH = HL::LPH, HPS = HL::HPS;
  const long long t = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  __nv_bfloat16* row = buf + t * ld;
  const int sub = lane % LPH, grp = lane / LPH;
  const bool act = sub < HL::CH;  // (always true unless dh = 80)
  float4 g[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)}, be[2] = {g[0], g[1]};
  if (act) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      g[i] = *reinterpret_cast<const float4*>(gamma + 8 * sub + 4 * i);
      be[i] = *reinterpret_cast<const float4*>(beta + 8 * sub + 4 * i);
    }
  }
  for (int base = 0; base < nheads; base += HPS) {
    const int hh = base + grp;  // (heads beyond nheads: the group only joins the shuffles)
    uint4 raw = act ? *(reinterpret_cast<const uint4*>(row + (hh < nheads ? hh : 0) * DH) + sub)
                    : make_uint4(0, 0, 0, 0);
    __nv_bfloat162* h2 = reinterpret_cast<__nv_bfloat162*>(&raw);
    float2 f[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) f[i] = __bfloat1622float2(h2[i]);
    float s1 = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) s1 += f[i].x + f[i].y;
#pragma unroll
    for (int o = LPH / 2; o > 0; o >>= 1) s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    const float mean = s1 * (1.0f / (float)DH);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[i].x -= mean;
      f[i].y -= mean;
      q = fmaf(f[i].x, f[i].x, fmaf(f[i].y, f[i].y, q));
    }
    if (!act) q = 0.f;  // dh 80: an idle lane's zeros would add (0 - mean)^2
#pragma unroll
    for (int o = LPH / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float inv = rsqrtf(q * (1.0f / (float)DH) + eps);
    if (hh < nheads && act) {
      const float gg[8] = {g[0].x, g[0].y, g[0].z, g[0].w, g[1].x, g[1].y, g[1].z, g[1].w};
      const float bb[8] = {be[0].x, be[0].y, be[0].z, be[0].w, be[1].x, be[1].y, be[1].z, be[1].w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float a = f[i].x * inv * gg[2 * i] + bb[2 * i], c = f[i].y * inv * gg[2 * i + 1] + bb[2 * i + 1];
        gelu_erf2(a, c);
        h2[i] = __floats2bfloat162_rn(a, c);
      }
      *(reinterpret_cast<uint4*>(row + hh * DH) + sub) = raw;
    }
  }
}

// NaViT attention pooling (reference na_vit.py:371-387): one learned query per image attends to that image's tokens.
//   kv[T, 2*H*DH] bf16 (k already RMS-normalised, then v), qn[H*DH] fp32 (normalised query), sequences by cu_seqlens;
//   out[S, H*DH] bf16 = softmax_j(qn_h . k_jh) v_jh   (scale 1).  One CTA of 8 warps per (image, head): warp w walks the
//   token groups w, w + 8, ... (4 tokens each) with an online softmax, the 8 partial (max, sum, acc) are merged in
//   shared memory -- a 1024-token image no longer takes 64x the time of a 16-token one on a single warp.
//   Lane l owns the element pairs l, l + 32, ... of the head (NP = DH / 64 rounded up); pairs beyond DH / 2 (dh 32
//   and 80) are masked: zero q, k and v, never stored.
//
// CLS = true: class-token cross attention (CrossViT, reference cross_vit.py:53-71 with kv_include_self): the query of
//   image s is row s of the packed qkv_self[S, 3*H*DH] (bf16, q | k | v), multiplied by `scale`; its own k and v (the
//   same row) are the first key and value, taken by warp 0 before its share of the context.  The n context [k | v]
//   rows of image s are rows s*ctx_rows + ctx_first + j (j < n) of kv, row stride ctx_ld; out row stride ldo.  cu and
//   qn are unused.  The CLS = false instances (NaViT) read none of the trailing parameters.
template <int DH, bool CLS = false>
__global__ void __launch_bounds__(256)
attn_pool_kernel(const __nv_bfloat16* __restrict__ kv, const float* __restrict__ qn, const int* __restrict__ cu,
                 __nv_bfloat16* __restrict__ out, int S, int H, const __nv_bfloat16* __restrict__ qkv_self = nullptr,
                 long long ctx_ld = 0, long long ctx_rows = 0, int ctx_first = 0, int n = 0, long long ldo = 0,
                 float scale = 1.f) {
  constexpr int NW = 8;
  constexpr int NP = (DH + 63) / 64;   // element pairs per lane
  __shared__ float part[NW][4 + DH];   // m, l, -, -, acc[DH]
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x / H, h = blockIdx.x % H;
  const int I = H * DH;
  bool act[NP];
  float2 q[NP];
  const __nv_bfloat16* self = CLS ? qkv_self + (long long)s * 3 * I + h * DH : nullptr;
#pragma unroll
  for (int c = 0; c < NP; ++c) {
    act[c] = 2 * (32 * c + lane) < DH;
    if (CLS) {
      const float2 z = make_float2(0.f, 0.f);
      const float2 qq = act[c] ? __bfloat1622float2(*(reinterpret_cast<const __nv_bfloat162*>(self) + 32 * c + lane)) : z;
      q[c] = make_float2(qq.x * scale, qq.y * scale);
    } else {
      q[c] = act[c] ? *reinterpret_cast<const float2*>(qn + h * DH + 2 * (32 * c + lane)) : make_float2(0.f, 0.f);
    }
  }
  float m = -INFINITY, l = 0.f, a0[NP], a1[NP];
#pragma unroll
  for (int c = 0; c < NP; ++c) a0[c] = a1[c] = 0.f;
  if (CLS && warp == 0) {
    // the query token's own key and value (kv_include_self, cross_vit.py:58-59) open warp 0's running softmax
    float sc = 0.f;
#pragma unroll
    for (int c = 0; c < NP; ++c) {
      if (!act[c]) continue;
      const float2 k = __bfloat1622float2(*(reinterpret_cast<const __nv_bfloat162*>(self + I) + 32 * c + lane));
      const float2 v = __bfloat1622float2(*(reinterpret_cast<const __nv_bfloat162*>(self + 2 * I) + 32 * c + lane));
      sc += q[c].x * k.x + q[c].y * k.y;
      a0[c] = v.x;
      a1[c] = v.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sc += __shfl_xor_sync(0xffffffffu, sc, o);
    m = sc;
    l = 1.f;
  }
  const int j0 = CLS ? 0 : cu[s], j1 = CLS ? n : cu[s + 1];
  const __nv_bfloat16* ctx = CLS ? kv + ((long long)s * ctx_rows + ctx_first) * ctx_ld + h * DH : nullptr;
  // four tokens per step: eight independent loads and four interleaved butterflies, one rescale of the running sums
  for (int j = j0 + 4 * warp; j < j1; j += 4 * NW) {
    const int cnt = j1 - j < 4 ? j1 - j : 4;
    float2 k[4][NP], v[4][NP];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const __nv_bfloat16* r = CLS ? ctx + (long long)(j + (i < cnt ? i : 0)) * ctx_ld
                                   : kv + (long long)(j + (i < cnt ? i : 0)) * 2 * I + h * DH;
#pragma unroll
      for (int c = 0; c < NP; ++c) {
        const float2 z = make_float2(0.f, 0.f);
        k[i][c] = act[c] ? __bfloat1622float2(*(reinterpret_cast<const __nv_bfloat162*>(r) + 32 * c + lane)) : z;
        v[i][c] = act[c] ? __bfloat1622float2(*(reinterpret_cast<const __nv_bfloat162*>(r + I) + 32 * c + lane)) : z;
      }
    }
    float sc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      sc[i] = q[0].x * k[i][0].x + q[0].y * k[i][0].y;
#pragma unroll
      for (int c = 1; c < NP; ++c) sc[i] += q[c].x * k[i][c].x + q[c].y * k[i][c].y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int i = 0; i < 4; ++i) sc[i] += __shfl_xor_sync(0xffffffffu, sc[i], o);
    }
#pragma unroll
    for (int i = 1; i < 4; ++i)
      if (i >= cnt) sc[i] = -INFINITY;         // tail group: the duplicated token 0 gets weight 0
    const float mn = fmaxf(fmaxf(m, fmaxf(sc[0], sc[1])), fmaxf(sc[2], sc[3]));
    const float corr = __expf(m - mn);
    l *= corr;
#pragma unroll
    for (int c = 0; c < NP; ++c) {
      a0[c] *= corr;
      a1[c] *= corr;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float pj = __expf(sc[i] - mn);
      l += pj;
#pragma unroll
      for (int c = 0; c < NP; ++c) {
        a0[c] = fmaf(pj, v[i][c].x, a0[c]);
        a1[c] = fmaf(pj, v[i][c].y, a1[c]);
      }
    }
    m = mn;
  }
  if (lane == 0) {
    part[warp][0] = m;
    part[warp][1] = l;
  }
#pragma unroll
  for (int c = 0; c < NP; ++c)
    if (act[c]) {
      part[warp][4 + 2 * (32 * c + lane)] = a0[c];
      part[warp][5 + 2 * (32 * c + lane)] = a1[c];
    }
  __syncthreads();
  if (warp == 0) {
    float mm = -INFINITY;
#pragma unroll
    for (int w = 0; w < NW; ++w) mm = fmaxf(mm, part[w][0]);
#pragma unroll
    for (int c = 0; c < NP; ++c) {
      if (!act[c]) continue;
      const int e = 2 * (32 * c + lane);
      float L = 0.f, A0 = 0.f, A1 = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        const float f = part[w][0] == -INFINITY ? 0.f : __expf(part[w][0] - mm);   // warps without a token
        L = fmaf(part[w][1], f, L);
        A0 = fmaf(part[w][4 + e], f, A0);
        A1 = fmaf(part[w][5 + e], f, A1);
      }
      const float inv = 1.0f / L;
      *reinterpret_cast<__nv_bfloat162*>(out + (long long)s * (CLS ? ldo : I) + h * DH + e) =
          __floats2bfloat162_rn(A0 * inv, A1 * inv);
    }
  }
}

// NaViT token assembly for packed variable-size images (reference na_vit.py:228,350-359): LayerNorm(dim, no bias) of
// the patch projection + factorised positional embedding pos_h[row] + pos_w[col] of the token's place in ITS image's
// patch grid -> fp32 residual stream, and (LN-fold entry) the bf16 copy + row statistics of it.  One warp per token;
// the image of a token is found by bisection of cu_seqlens, its grid width is dims[s][1] / p.
__global__ void __launch_bounds__(256)
embed_varlen_kernel(const float* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ pos_h,
                    const float* __restrict__ pos_w, const int* __restrict__ cu, const int* __restrict__ dims,
                    float* __restrict__ x, __nv_bfloat16* __restrict__ xb, float* __restrict__ stats, int T, int D,
                    int S, int p, float eps, int pos_h_rows, int pos_w_rows) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= T) return;
  int lo = 0, hi = S;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cu[mid] <= row) lo = mid; else hi = mid;
  }
  const int local = (int)row - cu[lo];
  // the host binding rejects grids larger than the tables (the reference raises an index error there); the clamps
  // only make sure a foreign caller of the C ABI can never read outside them
  const int gw = max(dims[2 * lo + 1] / p, 1);
  const float* ph = pos_h + (long long)min(local / gw, pos_h_rows - 1) * D;
  const float* pw = pos_w + (long long)min(local % gw, pos_w_rows - 1) * D;
  const float* yr = y + row * D;
  float* xr = x + row * D;
  __nv_bfloat16* xbr = xb ? xb + row * D : nullptr;
  float mean, rstd;
  ln_row_stats(yr, D, lane, mean, rstd, eps);
  // same association as the reference: (LN + pos_h) + pos_w.  D % 4 == 0 (checked by the launcher): only the float4
  // form runs.
  emit_row_stats<true>(
      D, lane, xr, xbr, stats ? stats + 2 * row : nullptr,
      [&](int i) {
        const float4 v = *reinterpret_cast<const float4*>(yr + i);
        const float4 g = *reinterpret_cast<const float4*>(gamma + i);
        const float4 a = *reinterpret_cast<const float4*>(ph + i);
        const float4 b = *reinterpret_cast<const float4*>(pw + i);
        return make_float4(((v.x - mean) * rstd * g.x + a.x) + b.x, ((v.y - mean) * rstd * g.y + a.y) + b.y,
                           ((v.z - mean) * rstd * g.z + a.z) + b.z, ((v.w - mean) * rstd * g.w + a.w) + b.w);
      },
      [&](int i) { return ((yr[i] - mean) * rstd * gamma[i] + ph[i]) + pw[i]; });
}

}  // namespace b200

// one launch of rmsnorm_heads_kernel<DH, U, LN> for a runtime dh (checked by the caller)
template <bool LN>
static void launch_heads_norm(__nv_bfloat16* b, int64_t ld, const float* gamma, int T, int nheads, int dh, float eps,
                              cudaStream_t st) {
  const dim3 grid((T + 7) / 8);
  const bool big = nheads > 8;
  switch (dh) {
    case 32:
      if (big) b200::rmsnorm_heads_kernel<32, 4, LN><<<grid, 256, 0, st>>>(b, ld, gamma, T, nheads, eps);
      else b200::rmsnorm_heads_kernel<32, 2, LN><<<grid, 256, 0, st>>>(b, ld, gamma, T, nheads, eps);
      break;
    case 80:
      if (big) b200::rmsnorm_heads_kernel<80, 4, LN><<<grid, 256, 0, st>>>(b, ld, gamma, T, nheads, eps);
      else b200::rmsnorm_heads_kernel<80, 2, LN><<<grid, 256, 0, st>>>(b, ld, gamma, T, nheads, eps);
      break;
    case 128:
      if (big) b200::rmsnorm_heads_kernel<128, 4, LN><<<grid, 256, 0, st>>>(b, ld, gamma, T, nheads, eps);
      else b200::rmsnorm_heads_kernel<128, 2, LN><<<grid, 256, 0, st>>>(b, ld, gamma, T, nheads, eps);
      break;
    default:
      if (big) b200::rmsnorm_heads_kernel<64, 4, LN><<<grid, 256, 0, st>>>(b, ld, gamma, T, nheads, eps);
      else b200::rmsnorm_heads_kernel<64, 2, LN><<<grid, 256, 0, st>>>(b, ld, gamma, T, nheads, eps);
  }
}

extern "C" int b200vit_layernorm_heads(void* buf, int64_t ld, const float* gamma, int T, int nheads, int dh, float eps,
                                       void* stream) {
  B200_CHECK_ARG(buf && gamma && T > 0 && nheads > 0, "layernorm_heads: bad argument");
  B200_CHECK_ARG(head_width_ok(dh), "layernorm_heads: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(ld >= (int64_t)nheads * dh && (ld % 8) == 0 && (reinterpret_cast<uintptr_t>(buf) & 15) == 0,
                 "layernorm_heads: rows must be 16-byte aligned and hold nheads*dh columns (ld=%lld)", (long long)ld);
  launch_heads_norm<true>(reinterpret_cast<__nv_bfloat16*>(buf), ld, gamma, T, nheads, dh, eps,
                          reinterpret_cast<cudaStream_t>(stream));
  B200_CHECK_CUDA(cudaGetLastError());
  b200::count_launch();
  return 0;
}

extern "C" int b200vit_head_layernorm_gelu(void* buf, int64_t ld, const float* gamma, const float* beta, int T,
                                           int nheads, int dh, float eps, void* stream) {
  B200_CHECK_ARG(buf && gamma && beta, "head_layernorm_gelu: null pointer");
  B200_CHECK_ARG(T > 0 && nheads > 0, "head_layernorm_gelu: bad shape T=%d nheads=%d", T, nheads);
  B200_CHECK_ARG(head_width_ok(dh), "head_layernorm_gelu: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(ld >= (int64_t)nheads * dh && (ld % 8) == 0 && (reinterpret_cast<uintptr_t>(buf) & 15) == 0,
                 "head_layernorm_gelu: rows must be 16-byte aligned and hold nheads*dh columns (ld=%lld)",
                 (long long)ld);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(gamma) & 15) == 0 && (reinterpret_cast<uintptr_t>(beta) & 15) == 0,
                 "head_layernorm_gelu: gamma and beta must be 16-byte aligned");
  auto* b = reinterpret_cast<__nv_bfloat16*>(buf);
  const dim3 grid((T + 7) / 8);
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: b200::head_layernorm_gelu_kernel<32><<<grid, 256, 0, st>>>(b, ld, gamma, beta, T, nheads, eps); break;
    case 80: b200::head_layernorm_gelu_kernel<80><<<grid, 256, 0, st>>>(b, ld, gamma, beta, T, nheads, eps); break;
    case 128: b200::head_layernorm_gelu_kernel<128><<<grid, 256, 0, st>>>(b, ld, gamma, beta, T, nheads, eps); break;
    default: b200::head_layernorm_gelu_kernel<64><<<grid, 256, 0, st>>>(b, ld, gamma, beta, T, nheads, eps);
  }
  B200_CHECK_CUDA(cudaGetLastError());
  b200::count_launch();
  return 0;
}

extern "C" int b200vit_rmsnorm_heads(void* buf, int64_t ld, const float* gamma, int T, int nheads, int dh,
                                     void* stream) {
  B200_CHECK_ARG(buf && gamma && T > 0 && nheads > 0, "rmsnorm_heads: bad argument");
  B200_CHECK_ARG(head_width_ok(dh), "rmsnorm_heads: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(ld >= (int64_t)nheads * dh && (ld % 8) == 0 && (reinterpret_cast<uintptr_t>(buf) & 15) == 0,
                 "rmsnorm_heads: rows must be 16-byte aligned and hold nheads*dh columns (ld=%lld)", (long long)ld);
  launch_heads_norm<false>(reinterpret_cast<__nv_bfloat16*>(buf), ld, gamma, T, nheads, dh, 0.f,
                           reinterpret_cast<cudaStream_t>(stream));
  B200_CHECK_CUDA(cudaGetLastError());
  b200::count_launch();
  return 0;
}

extern "C" int b200vit_qk_rmsnorm(void* qkv, const float* gamma_qk, int T, int H, int dh, void* stream) {
  B200_CHECK_ARG(qkv && gamma_qk && T > 0 && H > 0, "qk_rmsnorm: bad argument");
  B200_CHECK_ARG(head_width_ok(dh), "qk_rmsnorm: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  return b200vit_rmsnorm_heads(qkv, (int64_t)3 * H * dh, gamma_qk, T, 2 * H, dh, stream);  // q heads, then k heads
}

extern "C" int b200vit_embed_varlen(const float* y, const float* gamma, const float* pos_h, const float* pos_w,
                                    int pos_h_rows, int pos_w_rows, const int32_t* cu_seqlens_dev,
                                    const int32_t* dims_dev, float* x, void* xb_bf16, float* stats, int T, int D, int S,
                                    int p, float eps, void* stream) {
  B200_CHECK_ARG(y && gamma && pos_h && pos_w && cu_seqlens_dev && dims_dev && x, "embed_varlen: null pointer");
  B200_CHECK_ARG(pos_h_rows > 0 && pos_w_rows > 0, "embed_varlen: empty positional table");
  B200_CHECK_ARG(T > 0 && S > 0 && p > 0 && D > 0 && (D % 4) == 0, "embed_varlen: bad shape T=%d D=%d S=%d", T, D, S);
  b200::embed_varlen_kernel<<<(T + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      y, gamma, pos_h, pos_w, cu_seqlens_dev, dims_dev, x, reinterpret_cast<__nv_bfloat16*>(xb_bf16), stats, T, D, S, p,
      eps, pos_h_rows, pos_w_rows);
  B200_CHECK_CUDA(cudaGetLastError());
  b200::count_launch();
  return 0;
}

extern "C" int b200vit_attn_pool(const void* kv, const float* qn, const int32_t* cu_seqlens_dev, void* out, int S,
                                 int H, int dh, void* stream) {
  B200_CHECK_ARG(kv && qn && cu_seqlens_dev && out && S > 0 && H > 0, "attn_pool: bad argument");
  B200_CHECK_ARG(head_width_ok(dh), "attn_pool: dim_head=%d not supported by this build (32, 64, 80 or 128)", dh);
  const auto* k = reinterpret_cast<const __nv_bfloat16*>(kv);
  auto* o = reinterpret_cast<__nv_bfloat16*>(out);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: attn_pool_kernel<32><<<S * H, 256, 0, st>>>(k, qn, cu_seqlens_dev, o, S, H); break;
    case 80: attn_pool_kernel<80><<<S * H, 256, 0, st>>>(k, qn, cu_seqlens_dev, o, S, H); break;
    case 128: attn_pool_kernel<128><<<S * H, 256, 0, st>>>(k, qn, cu_seqlens_dev, o, S, H); break;
    default: attn_pool_kernel<64><<<S * H, 256, 0, st>>>(k, qn, cu_seqlens_dev, o, S, H);
  }
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200vit_attention_cls(const void* qkv_self, const void* ctx_kv, int64_t ctx_ld,
                                     int64_t ctx_rows_per_image, int ctx_first, int n, void* out, int64_t ldo, int B,
                                     int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(qkv_self && out && (ctx_kv || n == 0), "attention_cls: null pointer");
  B200_CHECK_ARG(B > 0 && H > 0, "attention_cls: bad shape B=%d H=%d", B, H);
  B200_CHECK_ARG(head_width_ok(dh) || dh == 48,
                 "attention_cls: dim_head=%d not supported by this build (32, 48, 64, 80 or 128)", dh);
  B200_CHECK_ARG(n >= 0 && n <= 16384, "attention_cls: n=%d context rows out of range [0, 16384]", n);
  B200_CHECK_ARG(ctx_first >= 0 && ctx_rows_per_image >= (int64_t)ctx_first + n,
                 "attention_cls: context rows [%d, %d) exceed the %lld rows per image", ctx_first, ctx_first + n,
                 (long long)ctx_rows_per_image);
  const int64_t I = (int64_t)H * dh;
  B200_CHECK_ARG(ldo >= I && (ldo % 8) == 0, "attention_cls: ldo=%lld must be >= H*dh and a multiple of 8",
                 (long long)ldo);
  B200_CHECK_ARG(n == 0 || (ctx_ld >= 2 * I && (ctx_ld % 8) == 0),
                 "attention_cls: ctx_ld=%lld must be >= 2*H*dh and a multiple of 8", (long long)ctx_ld);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv_self) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(ctx_kv) & 15) == 0,
                 "attention_cls: qkv_self, ctx_kv and out must be 16-byte aligned");
  B200_CHECK_ARG((int64_t)B * H <= 0x7fffffff, "attention_cls: B*H too large");
  const auto* q = reinterpret_cast<const __nv_bfloat16*>(qkv_self);
  const auto* k = reinterpret_cast<const __nv_bfloat16*>(ctx_kv);
  auto* o = reinterpret_cast<__nv_bfloat16*>(out);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  const long long ld = ctx_ld, rows = ctx_rows_per_image, lo = ldo;
  switch (dh) {
    case 32:
      attn_pool_kernel<32, true><<<B * H, 256, 0, st>>>(k, nullptr, nullptr, o, B, H, q, ld, rows, ctx_first, n, lo,
                                                        scale);
      break;
    case 48:
      attn_pool_kernel<48, true><<<B * H, 256, 0, st>>>(k, nullptr, nullptr, o, B, H, q, ld, rows, ctx_first, n, lo,
                                                        scale);
      break;
    case 80:
      attn_pool_kernel<80, true><<<B * H, 256, 0, st>>>(k, nullptr, nullptr, o, B, H, q, ld, rows, ctx_first, n, lo,
                                                        scale);
      break;
    case 128:
      attn_pool_kernel<128, true><<<B * H, 256, 0, st>>>(k, nullptr, nullptr, o, B, H, q, ld, rows, ctx_first, n, lo,
                                                         scale);
      break;
    default:
      attn_pool_kernel<64, true><<<B * H, 256, 0, st>>>(k, nullptr, nullptr, o, B, H, q, ld, rows, ctx_first, n, lo,
                                                        scale);
  }
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// NaViT patch extraction for a LIST of images of different sizes + LayerNorm(patch_dim, no bias), one launch:
//   out[cu[s] + h*gw_s + w, (c*p + p1)*p + p2] = LN_over_patch(img_s[c, h*p + p1, w*p + p2]) * gamma
// (reference na_vit.py:300 'c (h p1) (w p2) -> (h w) (c p1 p2)' + to_patch_embedding[0], na_vit.py:224-228,350).
// One CTA per patch row of one image (persistent): the C x p x W_s pixel slab is staged in shared memory with
// coalesced loads, then each warp normalises whole patches.  img_ptrs: device array of the images' data pointers.
// ---------------------------------------------------------------------------------------------------------------
namespace b200 {

__global__ void __launch_bounds__(256)
patchify_varlen_ln_kernel(const long long* __restrict__ img_ptrs, const int* __restrict__ dims,
                          const int* __restrict__ cu, const int* __restrict__ row_prefix,
                          const float* __restrict__ gamma, __nv_bfloat16* __restrict__ out, long long ldo, int S, int C,
                          int p, float eps) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* slab = reinterpret_cast<__nv_bfloat16*>(smem_raw);  // [C][p][W]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_rows = row_prefix[S];
  const int pd = C * p * p;
  for (int r = blockIdx.x; r < total_rows; r += gridDim.x) {
    int lo = 0, hi = S;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (row_prefix[mid] <= r) lo = mid; else hi = mid;
    }
    const int s = lo, h = r - row_prefix[s];
    const int H = dims[2 * s], W = dims[2 * s + 1];
    const int gw = W / p;
    const __nv_bfloat16* img = reinterpret_cast<const __nv_bfloat16*>(img_ptrs[s]);
    __syncthreads();  // previous slab fully consumed
    const int row_elems = p * W;
    for (int i = threadIdx.x; i < C * row_elems; i += blockDim.x) {
      const int c = i / row_elems, rr = i % row_elems;
      slab[i] = img[((long long)c * H + (long long)h * p) * W + rr];
    }
    __syncthreads();
    for (int w = warp; w < gw; w += 8) {
      // element e = (c*p + p1)*p + p2  <->  slab[(c*p + p1)*W + w*p + p2]
      float sum = 0.f;
      for (int e = lane; e < pd; e += 32) sum += __bfloat162float(slab[(e / p) * W + w * p + (e % p)]);
      const float mean = warp_sum(sum) / (float)pd;
      float q = 0.f;
      for (int e = lane; e < pd; e += 32) {
        const float d = __bfloat162float(slab[(e / p) * W + w * p + (e % p)]) - mean;
        q += d * d;
      }
      const float rstd = rsqrtf(warp_sum(q) / (float)pd + eps);
      __nv_bfloat16* orow = out + ((long long)cu[s] + (long long)h * gw + w) * ldo;
      for (int e = lane; e < (int)ldo; e += 32) {
        float y = 0.f;
        if (e < pd) y = (__bfloat162float(slab[(e / p) * W + w * p + (e % p)]) - mean) * rstd * gamma[e];
        orow[e] = __float2bfloat16_rn(y);
      }
    }
  }
}

// p == 16 fast path (C <= 4, out rows 16-byte aligned): the slab rows are padded by 16 bytes so that the 16-byte chunk
// reads of a patch (row stride W*2 bytes, often a multiple of 512) do not collide on banks; every lane owns C chunks of
// 8 pixels = one 16-byte piece of the output row, so the patch is read once, normalised in registers and written with
// fully coalesced 16-byte stores.  Images whose base is 16-byte aligned and whose width is a multiple of 8 are staged
// with 16-byte loads, others element by element.
__global__ void __launch_bounds__(256)
patchify_varlen_ln16_kernel(const long long* __restrict__ img_ptrs, const int* __restrict__ dims,
                            const int* __restrict__ cu, const int* __restrict__ row_prefix,
                            const float* __restrict__ gamma, __nv_bfloat16* __restrict__ out, long long ldo, int S,
                            int C, int wp, float eps) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* slab = reinterpret_cast<__nv_bfloat16*>(smem_raw);  // [C*16][wp]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_rows = row_prefix[S];
  const int pd = C * 256;
  const float inv_pd = 1.0f / (float)pd;
  for (int r = blockIdx.x; r < total_rows; r += gridDim.x) {
    int lo = 0, hi = S;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (row_prefix[mid] <= r) lo = mid; else hi = mid;
    }
    const int s = lo, h = r - row_prefix[s];
    const int H = dims[2 * s], W = dims[2 * s + 1];
    const int gw = W >> 4;
    const __nv_bfloat16* img = reinterpret_cast<const __nv_bfloat16*>(img_ptrs[s]);
    __syncthreads();  // previous slab fully consumed
    if (((W & 7) == 0) && ((reinterpret_cast<uintptr_t>(img) & 15) == 0)) {
      const int vpr = W >> 3;
      for (int i = threadIdx.x; i < C * 16 * vpr; i += blockDim.x) {
        const int rowi = i / vpr, vx = i - rowi * vpr;
        const int c = rowi >> 4, p1 = rowi & 15;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(img + ((long long)c * H + h * 16 + p1) * W) + vx);
        *(reinterpret_cast<uint4*>(slab + (long long)rowi * wp) + vx) = v;
      }
    } else {
      for (int i = threadIdx.x; i < C * 16 * W; i += blockDim.x) {
        const int rowi = i / W, xx = i - rowi * W;
        const int c = rowi >> 4, p1 = rowi & 15;
        slab[(long long)rowi * wp + xx] = img[((long long)c * H + h * 16 + p1) * W + xx];
      }
    }
    __syncthreads();
    for (int w = warp; w < gw; w += 8) {
      uint4 raw[4];
      float sum = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k < C) {
          const int j = lane + 32 * k;  // 16-byte chunk j of the patch: slab row j/2, half j%2
          raw[k] = *reinterpret_cast<const uint4*>(slab + (long long)(j >> 1) * wp + w * 16 + (j & 1) * 8);
          const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw[k]);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = __bfloat1622float2(h2[i]);
            sum += f.x + f.y;
          }
        }
      }
      const float mean = warp_sum(sum) * inv_pd;
      float q = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k < C) {
          const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw[k]);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = __bfloat1622float2(h2[i]);
            const float a = f.x - mean, b = f.y - mean;
            q = fmaf(a, a, fmaf(b, b, q));
          }
        }
      }
      const float rstd = rsqrtf(warp_sum(q) * inv_pd + eps);
      __nv_bfloat16* orow = out + ((long long)cu[s] + (long long)h * gw + w) * ldo;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k < C) {
          const int j = lane + 32 * k;
          const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw[k]);
          const float4 g0 = *reinterpret_cast<const float4*>(gamma + j * 8);
          const float4 g1 = *reinterpret_cast<const float4*>(gamma + j * 8 + 4);
          const float2 f0 = __bfloat1622float2(h2[0]), f1 = __bfloat1622float2(h2[1]);
          const float2 f2 = __bfloat1622float2(h2[2]), f3 = __bfloat1622float2(h2[3]);
          uint4 pk;
          pk.x = pack_bf16x2((f0.x - mean) * rstd * g0.x, (f0.y - mean) * rstd * g0.y);
          pk.y = pack_bf16x2((f1.x - mean) * rstd * g0.z, (f1.y - mean) * rstd * g0.w);
          pk.z = pack_bf16x2((f2.x - mean) * rstd * g1.x, (f2.y - mean) * rstd * g1.y);
          pk.w = pack_bf16x2((f3.x - mean) * rstd * g1.z, (f3.y - mean) * rstd * g1.w);
          *reinterpret_cast<uint4*>(orow + j * 8) = pk;
        }
      }
      for (int e = pd + lane; e < (int)ldo; e += 32) orow[e] = __float2bfloat16_rn(0.f);  // K padding of the GEMM operand
    }
  }
}

}  // namespace b200

extern "C" int b200vit_patchify_varlen_ln(const int64_t* img_ptrs_dev, const int32_t* dims_dev,
                                          const int32_t* cu_seqlens_dev, const int32_t* row_prefix_dev,
                                          const float* gamma, void* out_bf16, int64_t ldo, int S, int total_rows,
                                          int max_w, int C, int p, float eps, void* stream) {
  B200_CHECK_ARG(img_ptrs_dev && dims_dev && cu_seqlens_dev && row_prefix_dev && gamma && out_bf16,
                 "patchify_varlen_ln: null pointer");
  B200_CHECK_ARG(S > 0 && total_rows > 0 && C > 0 && p > 0 && max_w >= p, "patchify_varlen_ln: bad shape");
  B200_CHECK_ARG(ldo >= (int64_t)C * p * p, "patchify_varlen_ln: ldo too small");
  const bool fast = p == 16 && C <= 4 && (ldo % 8) == 0 && (reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0;
  const int wp = (max_w + 31) / 32 * 32 + 16;  // fast path: slab row stride in pixels (= 16 bytes mod 64: no bank conflicts)
  const size_t smem = fast ? (size_t)C * 16 * wp * 2 : (size_t)C * p * max_w * 2;
  B200_CHECK_ARG(smem <= 200 * 1024, "patchify_varlen_ln: patch-row slab of %zu bytes exceeds shared memory", smem);
  if (fast) B200_ENSURE_SMEM(b200::patchify_varlen_ln16_kernel, smem);
  else B200_ENSURE_SMEM(b200::patchify_varlen_ln_kernel, smem);
  int per_sm = (int)(200 * 1024 / (smem + 1024));
  if (per_sm > 8) per_sm = 8;
  if (per_sm < 1) per_sm = 1;
  int grid = b200::num_sms() * per_sm;
  if (grid > total_rows) grid = total_rows;
  auto st = reinterpret_cast<cudaStream_t>(stream);
  if (fast)
    b200::patchify_varlen_ln16_kernel<<<grid, 256, smem, st>>>(
        reinterpret_cast<const long long*>(img_ptrs_dev), dims_dev, cu_seqlens_dev, row_prefix_dev, gamma,
        reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, S, C, wp, eps);
  else
    b200::patchify_varlen_ln_kernel<<<grid, 256, smem, st>>>(
        reinterpret_cast<const long long*>(img_ptrs_dev), dims_dev, cu_seqlens_dev, row_prefix_dev, gamma,
        reinterpret_cast<__nv_bfloat16*>(out_bf16), ldo, S, C, p, eps);
  B200_CHECK_CUDA(cudaGetLastError());
  b200::count_launch();
  return 0;
}


// ------------------------------------------------------------------------------------------------------------------
// (sum, sum of squares) of the C x 16 x 16 bf16 pixels of every 16 x 16 patch: the LayerNorm statistics the TMA patch
// embedding folds into its epilogue (b200vit_patch_embed_tma).  One warp per patch; lane = pixel row of the patch
// (channel-major), 32 bytes per lane and row.
// ------------------------------------------------------------------------------------------------------------------
namespace b200 {
__global__ void __launch_bounds__(256)
patch_stats_kernel(const __nv_bfloat16* __restrict__ img, float* __restrict__ stats, long long num_patches, int C,
                   int H, int W) {
  const long long pidx = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (pidx >= num_patches) return;
  const int gw = W / 16, gh = H / 16;
  const int pw = (int)(pidx % gw), ph = (int)((pidx / gw) % gh);
  const long long b = pidx / ((long long)gw * gh);
  float s1 = 0.f, s2 = 0.f;
  for (int r = lane; r < C * 16; r += 32) {
    const int c = r >> 4, p1 = r & 15;
    const uint4* src = reinterpret_cast<const uint4*>(img + ((b * C + c) * H + ph * 16 + p1) * (long long)W + pw * 16);
    const uint4 v0 = src[0], v1 = src[1];
    const uint32_t w[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float lo = __uint_as_float(w[i] << 16), hi = __uint_as_float(w[i] & 0xFFFF0000u);
      s1 += lo + hi;
      s2 = fmaf(lo, lo, fmaf(hi, hi, s2));
    }
  }
  s1 = warp_sum(s1);
  s2 = warp_sum(s2);
  if (lane == 0) {
    stats[2 * pidx] = s1;
    stats[2 * pidx + 1] = s2;
  }
}
}  // namespace b200

extern "C" int b200vit_patch_stats(const void* img, float* stats, int B, int C, int H, int W, void* stream) {
  B200_CHECK_ARG(img && stats, "patch_stats: null pointer");
  B200_CHECK_ARG(B > 0 && C > 0 && (H % 16) == 0 && (W % 16) == 0 && H > 0 && W > 0,
                 "patch_stats: needs 16 x 16 patches on an image whose sides are multiples of 16");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(img) & 15) == 0, "patch_stats: image must be 16-byte aligned");
  const long long np = (long long)B * (H / 16) * (W / 16);
  b200::patch_stats_kernel<<<(unsigned)((np + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(img), stats, np, C, H, W);
  B200_CHECK_CUDA(cudaGetLastError());
  b200::count_launch();
  return 0;
}
