// vitron_b200 — RMSNorm / LayerNorm / GroupNorm(NHWC), HBM-bound, 16-byte vectorised, fp32 stats.
//   rmsnorm   : HF LlamaRMSNorm (transformers 4.31 modeling_llama.py, called per decoder layer)
//   layernorm : nn.LayerNorm of CLIPEncoderLayer (languagebind/image/modeling_image.py:136-151),
//               BasicTransformerBlock (i2vgen util.py:510-540), SEEM / GLIGEN blocks
//   groupnorm : nn.GroupNorm(32, C) (+SiLU) of ResBlock / TemporalConvBlock_v2 / transformers
//               (i2vgen util.py:640-655, 1358-1375, 1014) on NHWC [n, spatial, c] tensors
#include "common.cuh"
#include <cstdio>
#include "vitron_b200.h"

namespace vb {

template <int THREADS>
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (threadIdx.x < THREADS / 32) ? red[threadIdx.x] : 0.f;
  if (w == 0) {
    t = warp_sum(t);
    if (l == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

// one CTA per row; the row lives in registers between the statistics and the apply pass
template <int THREADS, int VPT, bool LAYER>
__global__ void __launch_bounds__(THREADS)
rownorm_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ w,
               const bf16* __restrict__ b, bf16* __restrict__ out, long long ldo, int d, float eps) {
  __shared__ float red[32];
  pdl_trigger();
  pdl_wait();
  const long long row = blockIdx.x;
  const bf16* xr = x + row * ldx;
  bf16* orow = out + row * ldo;
  float v[VPT * 8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = (i * THREADS + threadIdx.x) * 8;
    if (c < d) {
      uint4 u = *reinterpret_cast<const uint4*>(xr + c);
      float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
      v[i * 8 + 0] = f0.x; v[i * 8 + 1] = f0.y; v[i * 8 + 2] = f1.x; v[i * 8 + 3] = f1.y;
      v[i * 8 + 4] = f2.x; v[i * 8 + 5] = f2.y; v[i * 8 + 6] = f3.x; v[i * 8 + 7] = f3.y;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += LAYER ? v[i * 8 + j] : v[i * 8 + j] * v[i * 8 + j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i * 8 + j] = 0.f;
    }
  }
  float mean = 0.f, rstd;
  if (LAYER) {
    mean = block_sum<THREADS>(s, red) / d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = (i * THREADS + threadIdx.x) * 8;
      if (c < d) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { float t = v[i * 8 + j] - mean; q += t * t; }
      }
    }
    rstd = rsqrtf(block_sum<THREADS>(q, red) / d + eps);
  } else {
    rstd = rsqrtf(block_sum<THREADS>(s, red) / d + eps);
  }
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = (i * THREADS + threadIdx.x) * 8;
    if (c < d) {
      uint4 uw = *reinterpret_cast<const uint4*>(w + c);
      float wv[8];
      float2 t;
      t = unpack_bf16(uw.x); wv[0] = t.x; wv[1] = t.y;
      t = unpack_bf16(uw.y); wv[2] = t.x; wv[3] = t.y;
      t = unpack_bf16(uw.z); wv[4] = t.x; wv[5] = t.y;
      t = unpack_bf16(uw.w); wv[6] = t.x; wv[7] = t.y;
      float bv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (LAYER && b != nullptr) {
        uint4 ub = *reinterpret_cast<const uint4*>(b + c);
        t = unpack_bf16(ub.x); bv[0] = t.x; bv[1] = t.y;
        t = unpack_bf16(ub.y); bv[2] = t.x; bv[3] = t.y;
        t = unpack_bf16(ub.z); bv[4] = t.x; bv[5] = t.y;
        t = unpack_bf16(ub.w); bv[6] = t.x; bv[7] = t.y;
      }
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[i * 8 + j] - mean) * rstd * wv[j] + bv[j];
      *reinterpret_cast<uint4*>(orow + c) = make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]),
                                                       pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7]));
    }
  }
}

// out[row] = rsqrt(mean(x^2) + eps): one warp per row
__global__ void row_rstd_kernel(const bf16* __restrict__ x, long long ldx, float* __restrict__ out, long long rows,
                                int d, float eps) {
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const bf16* xr = x + row * ldx;
  float s = 0.f;
  for (int c = lane * 8; c < d; c += 256) {
    const uint4 u = *reinterpret_cast<const uint4*>(xr + c);
    float2 f;
    f = unpack_bf16(u.x); s += f.x * f.x + f.y * f.y;
    f = unpack_bf16(u.y); s += f.x * f.x + f.y * f.y;
    f = unpack_bf16(u.z); s += f.x * f.x + f.y * f.y;
    f = unpack_bf16(u.w); s += f.x * f.x + f.y * f.y;
  }
  s = warp_sum(s);
  if (lane == 0) out[row] = rsqrtf(s / d + eps);
}

// d <= 1024: one WARP per row (8 rows per CTA); each lane keeps up to 4 x 8 elements in registers.
template <bool LAYER>
__global__ void __launch_bounds__(256)
rownorm_warp_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ w, const bf16* __restrict__ b,
                    bf16* __restrict__ out, long long ldo, long long rows, int d, float eps) {
  pdl_trigger();
  pdl_wait();
  const long long row = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const bf16* xr = x + row * ldx;
  float v[4][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = (i * 32 + lane) * 8;
    if (c < d) {
      const uint4 u = *reinterpret_cast<const uint4*>(xr + c);
      const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) { float2 f = unpack_bf16(uu[j]); v[i][2 * j] = f.x; v[i][2 * j + 1] = f.y; }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += LAYER ? v[i][j] : v[i][j] * v[i][j];
    }
  }
  s = warp_sum(s);
  float mean = 0.f, rstd;
  if (LAYER) {
    mean = s / d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = (i * 32 + lane) * 8;
      if (c < d) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float t = v[i][j] - mean; q += t * t; }
      }
    }
    rstd = rsqrtf(warp_sum(q) / d + eps);
  } else {
    rstd = rsqrtf(s / d + eps);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = (i * 32 + lane) * 8;
    if (c < d) {
      const uint4 uw = *reinterpret_cast<const uint4*>(w + c);
      const uint32_t ww[4] = {uw.x, uw.y, uw.z, uw.w};
      uint32_t bb[4] = {0, 0, 0, 0};
      if (LAYER && b != nullptr) {
        const uint4 ub = *reinterpret_cast<const uint4*>(b + c);
        bb[0] = ub.x; bb[1] = ub.y; bb[2] = ub.z; bb[3] = ub.w;
      }
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 wf = unpack_bf16(ww[j]), bf = unpack_bf16(bb[j]);
        o[j] = pack_bf16((v[i][2 * j] - mean) * rstd * wf.x + bf.x, (v[i][2 * j + 1] - mean) * rstd * wf.y + bf.y);
      }
      *reinterpret_cast<uint4*>(out + row * ldo + c) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// d <= 512 and many rows (UNet / ViT token LayerNorms): one warp per FOUR rows. All eight 16-byte loads of a
// lane are issued before the first reduction, the four shuffle chains interleave, and the gain / bias
// vectors are fetched once per warp instead of once per row.
template <bool LAYER>
__global__ void __launch_bounds__(256)
rownorm_warp4_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ w, const bf16* __restrict__ b,
                     bf16* __restrict__ out, long long ldo, long long rows, int d, float eps) {
  pdl_trigger();
  pdl_wait();
  const long long row0 = (blockIdx.x * 8LL + (threadIdx.x >> 5)) * 4;
  if (row0 >= rows) return;
  const int lane = threadIdx.x & 31;
  const int c0 = lane * 8, c1 = (32 + lane) * 8;
  const bool h0 = c0 < d, h1 = c1 < d;
  uint4 u[4][2];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const bool ok = row0 + r < rows;
    const bf16* xr = x + (row0 + r) * ldx;
    u[r][0] = (ok && h0) ? __ldg(reinterpret_cast<const uint4*>(xr + c0)) : make_uint4(0u, 0u, 0u, 0u);
    u[r][1] = (ok && h1) ? __ldg(reinterpret_cast<const uint4*>(xr + c1)) : make_uint4(0u, 0u, 0u, 0u);
  }
  float wv[2][8], bv[2][8];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int c = i ? c1 : c0;
    const bool has = i ? h1 : h0;
    uint4 uw = make_uint4(0u, 0u, 0u, 0u), ub = make_uint4(0u, 0u, 0u, 0u);
    if (has) {
      uw = __ldg(reinterpret_cast<const uint4*>(w + c));
      if (LAYER && b != nullptr) ub = __ldg(reinterpret_cast<const uint4*>(b + c));
    }
    const uint32_t ww[4] = {uw.x, uw.y, uw.z, uw.w}, bb[4] = {ub.x, ub.y, ub.z, ub.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 wf = unpack_bf16(ww[j]), bf = unpack_bf16(bb[j]);
      wv[i][2 * j] = wf.x; wv[i][2 * j + 1] = wf.y; bv[i][2 * j] = bf.x; bv[i][2 * j + 1] = bf.y;
    }
  }
  float v[4][2][8], s[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    s[r] = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t uu[4] = {u[r][i].x, u[r][i].y, u[r][i].z, u[r][i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float2 f = unpack_bf16(uu[j]); v[r][i][2 * j] = f.x; v[r][i][2 * j + 1] = f.y; }
#pragma unroll
      for (int j = 0; j < 8; ++j) s[r] += LAYER ? v[r][i][j] : v[r][i][j] * v[r][i][j];  // absent pieces are zero
    }
  }
#pragma unroll
  for (int sh = 16; sh > 0; sh >>= 1)
#pragma unroll
    for (int r = 0; r < 4; ++r) s[r] += __shfl_xor_sync(0xffffffffu, s[r], sh);
  float mean[4] = {0.f, 0.f, 0.f, 0.f}, rstd[4];
  if (LAYER) {
    float q[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      mean[r] = s[r] / d;
      q[r] = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (h0) { const float t = v[r][0][j] - mean[r]; q[r] += t * t; }
        if (h1) { const float t = v[r][1][j] - mean[r]; q[r] += t * t; }
      }
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1)
#pragma unroll
      for (int r = 0; r < 4; ++r) q[r] += __shfl_xor_sync(0xffffffffu, q[r], sh);
#pragma unroll
    for (int r = 0; r < 4; ++r) rstd[r] = rsqrtf(q[r] / d + eps);
  } else {
#pragma unroll
    for (int r = 0; r < 4; ++r) rstd[r] = rsqrtf(s[r] / d + eps);
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    if (row0 + r >= rows) break;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (!(i ? h1 : h0)) continue;
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        o[j] = pack_bf16((v[r][i][2 * j] - mean[r]) * rstd[r] * wv[i][2 * j] + bv[i][2 * j],
                         (v[r][i][2 * j + 1] - mean[r]) * rstd[r] * wv[i][2 * j + 1] + bv[i][2 * j + 1]);
      *reinterpret_cast<uint4*>(out + (row0 + r) * ldo + (i ? c1 : c0)) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <bool LAYER>
static int launch_rownorm(const void* x, long long ldx, const void* w, const void* b, void* out,
                          long long ldo, long long rows, long long d, float eps, cudaStream_t st) {
  if (rows <= 0) return VB_OK;
  if (d % 8 != 0 || ldx % 8 != 0 || ldo % 8 != 0) return VB_ERR_ARG;
  if (!aligned16(x) || !aligned16(w) || !aligned16(b) || !aligned16(out)) return VB_ERR_ARG;
  const bf16* xp = reinterpret_cast<const bf16*>(x);
  const bf16* wp = reinterpret_cast<const bf16*>(w);
  const bf16* bp = reinterpret_cast<const bf16*>(b);
  bf16* op = reinterpret_cast<bf16*>(out);
  unsigned grid = static_cast<unsigned>(rows);
  if (d <= 512 && rows >= 1024)
    vb_launch(rownorm_warp4_kernel<LAYER>, dim3(static_cast<unsigned>((rows + 31) / 32)), dim3(256), 0, st, xp, ldx, wp, bp, op, ldo, rows, (int)d, eps);
  else if (d <= 1024 && rows >= 64)
    vb_launch(rownorm_warp_kernel<LAYER>, dim3(static_cast<unsigned>((rows + 7) / 8)), dim3(256), 0, st, xp, ldx, wp, bp, op, ldo, rows, (int)d, eps);
  else if (d <= 128 * 8) vb_launch(rownorm_kernel<128, 1, LAYER>, dim3(grid), dim3(128), 0, st, xp, ldx, wp, bp, op, ldo, (int)d, eps);
  else if (d <= 256 * 8 * 1) vb_launch(rownorm_kernel<256, 1, LAYER>, dim3(grid), dim3(256), 0, st, xp, ldx, wp, bp, op, ldo, (int)d, eps);
  else if (d <= 256 * 8 * 2) vb_launch(rownorm_kernel<256, 2, LAYER>, dim3(grid), dim3(256), 0, st, xp, ldx, wp, bp, op, ldo, (int)d, eps);
  else if (d <= 256 * 8 * 4) vb_launch(rownorm_kernel<256, 4, LAYER>, dim3(grid), dim3(256), 0, st, xp, ldx, wp, bp, op, ldo, (int)d, eps);
  else if (d <= 512 * 8 * 4) vb_launch(rownorm_kernel<512, 4, LAYER>, dim3(grid), dim3(512), 0, st, xp, ldx, wp, bp, op, ldo, (int)d, eps);
  else return VB_ERR_UNSUPPORTED;
  VB_LAUNCH_CHECK();
  return VB_OK;
}

// ------------------------------------------------------------------ GroupNorm NHWC
// x: [n, spatial, c] bf16, group = channel / (c / groups). ONE launch, x read from global ONCE:
//
//   The grid is at most one CTA per SM and every CTA owns a contiguous slab of rows of ONE sample. Phase 1 streams
//   the slab with fully coalesced 16-byte loads (a thread owns one fixed 8-channel vector) INTO SHARED MEMORY
//   (up to ~190 KB per SM: the 26 MB level-0 UNet tensor is 177 KB per SM) while accumulating per-channel sums in
//   registers; the CTA folds them into per-group sums (smem, warp shuffles) and adds them to sums[n][groups][2] with
//   fp32 atomics. The CTAs of a sample then meet at a counter barrier (all CTAs are co-resident: grid <= SMs), every
//   CTA derives the per-channel affine (rstd*gamma, beta - mean*rstd*gamma) into smem, and phase 2 normalises its
//   slab OUT OF SHARED MEMORY with 16-byte stores. The last CTA to have read the sums zeroes the workspace again
//   (zero at allocation, left zero: no memset, stateless). Slabs beyond the smem budget (78 MB decoder concats) are
//   re-read from global (L2) in phase 2 by the same kernel.
//
//   History: round 1 = single-pass kernel over [spatial x 40-channel] slabs (80-byte row fragments) or stats + apply
//   kernels, 3.5 ms of a 25 ms UNet forward; a coalesced stats / apply pair with a last-CTA finaliser measured 15.7 +
//   16.6 us per GroupNorm — both launches are latency chains (launch, L2 round trips, atomics, fence) longer than
//   the data movement, so the fix is one launch and one read, not faster loops.
// Two sets of sums per channel: of x and x^2 (s, q), and of d = x - K and d^2 (ds, dq) around a pivot K per (sample,
// group), the group's first channel in the sample's first row. var = E[x^2] - mean^2 cancels in fp32 when the group mean
// is large next to its spread (at |mean| / std = 256, rstd came out 2e-2 off); var = E[d^2] - E[d]^2 does not. The
// statistics take the plain sums when |mean| <= 2 std and the pivot sums otherwise (gn_stats).
__device__ __forceinline__ void gn_accumulate(const uint4 u, const float (&k)[8], float (&s)[8], float (&q)[8],
                                              float (&ds)[8], float (&dq)[8]) {
  const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16(uu[j]);
    s[2 * j] += f.x; q[2 * j] += f.x * f.x; s[2 * j + 1] += f.y; q[2 * j + 1] += f.y * f.y;
    const float d0 = f.x - k[2 * j], d1 = f.y - k[2 * j + 1];
    ds[2 * j] += d0; dq[2 * j] += d0 * d0; ds[2 * j + 1] += d1; dq[2 * j + 1] += d1 * d1;
  }
}

// (mean, rstd) of a group from its plain sums (sum, sq) and its pivot sums (dsum, dsq) around k over cnt elements
__device__ __forceinline__ float2 gn_stats(float sum, float sq, float dsum, float dsq, float k, float cnt, float eps) {
  const float mean = sum / cnt;
  const float dm = dsum / cnt;
  const float dvar = fmaxf(dsq / cnt - dm * dm, 0.f);
  // (__fmul_rn: the test must not change how the plain formula below is contracted)
  if (__fmul_rn(mean, mean) > 4.f * dvar) return make_float2(k + dm, rsqrtf(dvar + eps));
  const float rstd = rsqrtf(fmaxf(sq / cnt - mean * mean, 0.f) + eps);
  return make_float2(mean, rstd);
}

// The CTAs of a sample publish their group partial sums in slots of their own (no atomics) and every CTA adds the slots
// of its sample in one fixed order, so the statistics — and everything downstream of them — are bit-identical from run
// to run.
struct GnWs {
  float* sums;      // [n * ctas per sample][groups][4]: one slot per CTA, overwritten by every launch
  int* arrived;     // [n]  CTAs of the sample that published their sums
  int* readers;     // [n]  CTAs of the sample that consumed the sums (the last one resets both counters)
};

// SiLU with ONE MUFU op per element: x * sigmoid(x) = 0.5 x (1 + tanh(x / 2)); tanh.approx.f32 has ~2^-11 relative error,
// below the bf16 rounding of the result. (x / (1 + exp(-x)) costs two — ex2 and rcp — and the 13 M-element level-0
// GroupNorms of the UNet were MUFU-bound on it: 186 k MUFU ops per SM at 16 per clock.)
__device__ __forceinline__ float silu_tanh(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * x));
  return fmaf(0.5f * x, t, 0.5f * x);
}

template <int ACT>
__device__ __forceinline__ uint4 gn_affine(const uint4 u, const float (&sc)[8], const float (&sh)[8]) {
  const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
  uint32_t oo[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16(uu[j]);
    float y0 = fmaf(f.x, sc[2 * j], sh[2 * j]);
    float y1 = fmaf(f.y, sc[2 * j + 1], sh[2 * j + 1]);
    if (ACT == VB_ACT_SILU) { y0 = silu_tanh(y0); y1 = silu_tanh(y1); }
    else if (ACT == VB_ACT_RELU) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
    oo[j] = pack_bf16(y0, y1);
  }
  return make_uint4(oo[0], oo[1], oo[2], oo[3]);
}

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// grid = (ctas_per_sample, n); blockDim = round_up32((c / 8) * rpp) (threads beyond (c/8)*rpp only take part in the
// barriers / shuffles); dynamic smem = [part: rpp*c*2 floats | slab: rows*c bf16 if CACHED]
template <int ACT, bool CACHED>
__global__ void __launch_bounds__(512)
gn_onepass_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, const bf16* __restrict__ b, bf16* __restrict__ out,
                  GnWs ws, int spatial, int c, int groups, int rows_per_cta, int rpp, float eps) {
  extern __shared__ __align__(128) uint8_t gsm[];
  __shared__ float gsum[1024];                                                        // [groups][2]: sums, then (mean, rstd)
  __shared__ float gpiv[512];                                                         // [groups] pivots
  __shared__ __align__(8) uint64_t slab_bar;
  float* part = reinterpret_cast<float*>(gsm);                                        // [rpp][c][2], later aff[2][c]
  uint4* slab = reinterpret_cast<uint4*>(gsm + static_cast<size_t>(rpp) * c * 2 * sizeof(float));  // [rows][c/8]
  const int n = blockIdx.y;
  const int vec_per_row = c >> 3;
  const bool active = threadIdx.x < vec_per_row * rpp;
  const int my_vec = threadIdx.x % vec_per_row, my_row = threadIdx.x / vec_per_row;
  const int r0 = blockIdx.x * rows_per_cta;
  const int rows = min(rows_per_cta, spatial - r0);
  const size_t off = (static_cast<size_t>(n) * spatial + r0) * c + my_vec * 8;
  const bf16* xb = x + off;
  pdl_trigger();
  if (CACHED && threadIdx.x == 0) {
    mbar_init(&slab_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // nothing of the predecessor's output has been touched above
  if (CACHED && threadIdx.x == 0) {
    // the CTA's slab is ONE contiguous range of global memory: the TMA unit copies it into shared memory in 32 KB
    // pieces (all in flight at once: the register-load loop this replaces kept ~30 KB per SM in flight and was latency
    // bound), every thread then accumulates its fixed 8-channel column out of shared memory
    const uint32_t total = static_cast<uint32_t>(rows) * c * 2;
    mbar_arrive_expect_tx(&slab_bar, total);
    const uint8_t* src = reinterpret_cast<const uint8_t*>(x + (static_cast<size_t>(n) * spatial + r0) * c);
    for (uint32_t o = 0; o < total; o += 32768) bulk_copy_g2s(reinterpret_cast<uint8_t*>(slab) + o, src + o, min(32768u, total - o), &slab_bar);
  }
  const int cpg = c / groups;
  const bf16* xn = x + static_cast<size_t>(n) * spatial * c;   // row 0 of the sample: the group pivots
  float s[8], q[8], ds[8], dq[8], kp[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s[j] = q[j] = ds[j] = dq[j] = 0.f;
    kp[j] = active ? __bfloat162float(xn[(my_vec * 8 + j) / cpg * cpg]) : 0.f;
  }
  // the statistics need the pivots again; read them now, before any CTA of the sample can overwrite row 0 (in place)
  for (int g = threadIdx.x; g < groups; g += blockDim.x) gpiv[g] = __bfloat162float(xn[g * cpg]);
  if (CACHED) {
    mbar_wait(&slab_bar, 0);
    if (active)
      for (int r = my_row; r < rows; r += rpp) gn_accumulate(slab[r * vec_per_row + my_vec], kp, s, q, ds, dq);
  } else if (active) {
    int r = my_row;
    for (; r + 7 * rpp < rows; r += 8 * rpp) {  // eight independent 16-byte loads in flight
      uint4 u[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(xb + static_cast<size_t>(r + k * rpp) * c));
#pragma unroll
      for (int k = 0; k < 8; ++k) gn_accumulate(u[k], kp, s, q, ds, dq);
    }
    for (; r < rows; r += rpp) gn_accumulate(__ldg(reinterpret_cast<const uint4*>(xb + static_cast<size_t>(r) * c)), kp, s, q, ds, dq);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;  // blockDim is a multiple of 32
  const int ctas = gridDim.x;
  const float cnt = static_cast<float>(cpg) * static_cast<float>(spatial);
  const float* gs = ws.sums + static_cast<size_t>(n) * ctas * groups * 4;           // the slots of this sample
  float* gs_mine = ws.sums + (static_cast<size_t>(n) * ctas + blockIdx.x) * groups * 4;  // this CTA's slot [groups][4]
  // the CTA's group sums, plain (pass 0) then pivot (pass 1), through the same [rpp][c][2] staging area; a group's sums are
  // reduced by the same warp in both passes, so with one CTA per sample its lane 0 holds all four and stores (mean, rstd)
  for (int pass = 0; pass < 2; ++pass) {
    if (active) {
      float* mine = part + (static_cast<size_t>(my_row) * c + my_vec * 8) * 2;
#pragma unroll
      for (int j = 0; j < 8; j += 2)
        *reinterpret_cast<float4*>(mine + j * 2) = pass == 0 ? make_float4(s[j], q[j], s[j + 1], q[j + 1])
                                                             : make_float4(ds[j], dq[j], ds[j + 1], dq[j + 1]);
    }
    __syncthreads();
    for (int g = warp; g < groups; g += nwarps) {
      float as = 0.f, aq = 0.f;
      const int items = rpp * cpg;
      for (int e = lane; e < items; e += 32) {
        const int rr = e / cpg, ch = g * cpg + (e - rr * cpg);
        const float2 v = *reinterpret_cast<const float2*>(part + (static_cast<size_t>(rr) * c + ch) * 2);
        as += v.x;
        aq += v.y;
      }
      as = warp_sum(as);
      aq = warp_sum(aq);
      if (lane == 0) {
        if (ctas > 1) {
          gs_mine[g * 4 + 2 * pass] = as;
          gs_mine[g * 4 + 2 * pass + 1] = aq;
        } else if (pass == 0) {  // the whole sample is this CTA: no global round trip
          gsum[g * 2] = as;
          gsum[g * 2 + 1] = aq;
        } else {
          const float2 st = gn_stats(gsum[g * 2], gsum[g * 2 + 1], as, aq, gpiv[g], cnt, eps);
          gsum[g * 2] = st.x;
          gsum[g * 2 + 1] = st.y;
        }
      }
    }
    __syncthreads();   // pass 1 overwrites the staging area
  }
  // ---- the CTAs of this sample meet: publish, then wait until all have published
  if (ctas > 1) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      atomicAdd(ws.arrived + n, 1);
      while (ld_acquire_gpu(ws.arrived + n) < ctas) { }
    }
  }
  __syncthreads();
  // ---- group sums of the sample = sum of its CTAs' slots, in a fixed order (lane l adds slots l, l + 32, ..., then a
  // fixed shuffle tree) -> (mean, rstd) in gsum; then the per-channel affine into smem (`part` is free: every warp passed
  // the barrier above after its reads)
  if (ctas > 1) {
    for (int g = warp; g < groups; g += nwarps) {
      float a[4] = {0.f, 0.f, 0.f, 0.f};
      for (int k = lane; k < ctas; k += 32) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(gs + (static_cast<size_t>(k) * groups + g) * 4));
        a[0] += v.x; a[1] += v.y; a[2] += v.z; a[3] += v.w;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = warp_sum(a[i]);
      if (lane == 0) {
        const float2 st = gn_stats(a[0], a[1], a[2], a[3], gpiv[g], cnt, eps);
        gsum[g * 2] = st.x;
        gsum[g * 2 + 1] = st.y;
      }
    }
    __syncthreads();
  }
  float* aff = part;  // [2][c]
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    const int g = ch / cpg;
    const float mean = gsum[g * 2], rstd = gsum[g * 2 + 1];
    const float sc = rstd * __bfloat162float(w[ch]);
    aff[ch] = sc;
    aff[c + ch] = __bfloat162float(b[ch]) - mean * sc;
  }
  __syncthreads();
  float sc[8], sh[8];
  {
    const float4 a0 = *reinterpret_cast<const float4*>(aff + my_vec * 8), a1 = *reinterpret_cast<const float4*>(aff + my_vec * 8 + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(aff + c + my_vec * 8), b1 = *reinterpret_cast<const float4*>(aff + c + my_vec * 8 + 4);
    sc[0] = a0.x; sc[1] = a0.y; sc[2] = a0.z; sc[3] = a0.w; sc[4] = a1.x; sc[5] = a1.y; sc[6] = a1.z; sc[7] = a1.w;
    sh[0] = b0.x; sh[1] = b0.y; sh[2] = b0.z; sh[3] = b0.w; sh[4] = b1.x; sh[5] = b1.y; sh[6] = b1.z; sh[7] = b1.w;
  }
  bf16* ob = out + off;
  if (!active) return;   // (thread 0 is always active)
  if (CACHED) {
    for (int rr = my_row; rr < rows; rr += rpp)
      *reinterpret_cast<uint4*>(ob + static_cast<size_t>(rr) * c) = gn_affine<ACT>(slab[rr * vec_per_row + my_vec], sc, sh);
  } else {
    int rr = my_row;
    for (; rr + 7 * rpp < rows; rr += 8 * rpp) {
      uint4 u[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(xb + static_cast<size_t>(rr + k * rpp) * c));
#pragma unroll
      for (int k = 0; k < 8; ++k)
        *reinterpret_cast<uint4*>(ob + static_cast<size_t>(rr + k * rpp) * c) = gn_affine<ACT>(u[k], sc, sh);
    }
    for (; rr < rows; rr += rpp)
      *reinterpret_cast<uint4*>(ob + static_cast<size_t>(rr) * c) =
          gn_affine<ACT>(__ldg(reinterpret_cast<const uint4*>(xb + static_cast<size_t>(rr) * c)), sc, sh);
  }
  if (ctas > 1 && threadIdx.x == 0) {
    // every thread of this CTA read the sums before the affine barrier: the last CTA of the sample to get here hands the
    // counters back zeroed (done after this thread's share of the apply pass so that it delays nothing)
    __threadfence();
    const int prev = atomicAdd(ws.readers + n, 1);
    if (prev == ctas - 1) {
      ws.arrived[n] = 0;
      ws.readers[n] = 0;
    }
  }
}

}  // namespace vb

using namespace vb;

extern "C" int vb200_rmsnorm(const void* x, int64_t ldx, const void* weight, void* out, int64_t ldo,
                             int64_t rows, int64_t d, float eps, cudaStream_t stream) {
  VB_CHECK_ARG(x && weight && out && d > 0);
  return launch_rownorm<false>(x, ldx, weight, nullptr, out, ldo, rows, d, eps, stream);
}

extern "C" int vb200_row_rstd(const void* x, int64_t ldx, float* out, int64_t rows, int64_t d, float eps,
                              cudaStream_t stream) {
  VB_CHECK_ARG(x && out && rows >= 0 && d > 0 && d % 8 == 0 && ldx % 8 == 0 && aligned16(x));
  if (rows == 0) return VB_OK;
  row_rstd_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, stream>>>(reinterpret_cast<const bf16*>(x), ldx, out,
                                                                             rows, static_cast<int>(d), eps);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_layernorm(const void* x, int64_t ldx, const void* weight, const void* bias,
                               void* out, int64_t ldo, int64_t rows, int64_t d, float eps,
                               cudaStream_t stream) {
  VB_CHECK_ARG(x && weight && out && d > 0);
  return launch_rownorm<true>(x, ldx, weight, bias, out, ldo, rows, d, eps, stream);
}

constexpr int GN_DYN_SMEM_MAX = 220 * 1024;  // dynamic smem budget of gn_onepass_kernel (+ 6 KB static <= 227 KB)

static size_t gn_align16(size_t v) { return (v + 15) & ~static_cast<size_t>(15); }

// The counters live in a FIXED-size prefix, the per-CTA sum slots behind it: one workspace serves calls of any n / groups
// without a call's counters ever landing on another call's (stale) sums. Larger batches run in chunks of GN_MAX_N samples.
constexpr int64_t GN_MAX_N = 1024;
constexpr size_t GN_COUNTER_BYTES = 2 * GN_MAX_N * sizeof(int);   // arrived[GN_MAX_N] | readers[GN_MAX_N]

extern "C" size_t vb200_groupnorm_workspace_size(int64_t n, int64_t groups, int64_t c) {
  // [arrival counters | reader counters | per-CTA group sums]; zero-fill ONCE before first use, the kernel leaves the
  // counters zeroed and overwrites the sum slots it reads (a launch has at most max(n, SM count) CTAs: gn_plan)
  (void)c;
  if (n > GN_MAX_N) n = GN_MAX_N;
  const int64_t ctas = n > vb_num_sms() ? n : vb_num_sms();
  return GN_COUNTER_BYTES + gn_align16(static_cast<size_t>(ctas) * groups * 4 * sizeof(float));
}

template <int ACT, bool CACHED>
static int gn_launch(const bf16* x, const bf16* w, const bf16* b, bf16* out, GnWs ws, int spatial, int c, int groups, int rpc,
                     int rpp, float eps, dim3 grid, int threads, size_t smem, cudaStream_t stream) {
  auto kern = gn_onepass_kernel<ACT, CACHED>;
  static bool attr_set = false;
  if (!attr_set) {
    // opt in once per instantiation, whatever the first launch needs: the default limit of 48 KB counts the kernel's 4 KB of
    // STATIC shared memory too (a first launch with exactly 48 KB of dynamic smem failed with "invalid argument").
    // 227 KB per CTA minus the static part (gsum + pivots + barrier: 6 KB)
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GN_DYN_SMEM_MAX);
    if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
    attr_set = true;
  }
  cudaError_t le = vb_launch(kern, grid, dim3(threads), smem, stream, x, w, b, out, ws, spatial, c, groups, rpc, rpp, eps);
  if (le != cudaSuccess) {
    fprintf(stderr, "vb200_groupnorm_nhwc launch failed (%s): grid (%u, %u) threads %d smem %zu cached %d spatial %d c %d groups %d rpc %d rpp %d\n",
            cudaGetErrorString(le), grid.x, grid.y, threads, smem, CACHED ? 1 : 0, spatial, c, groups, rpc, rpp);
    (void)cudaGetLastError();   // the failed launch must not be reported again by the next kernel's check
    vb_set_last_error(le);
    return VB_ERR_CUDA;
  }
  return VB_OK;
}

struct GnPlan {
  int rpp, threads;
  long long per, rpc;
  bool cached;
  size_t smem;
};

// launch shape of gn_onepass_kernel for n samples of spatial x c: CTAs per sample, rows per CTA, whether the CTA slab is cached
static GnPlan gn_plan(int64_t n, int64_t spatial, int64_t c) {
  GnPlan p;
  const int vec_per_row = static_cast<int>(c / 8);
  int rpp = 512 / vec_per_row;
  if (rpp < 1) rpp = 1;
  if (rpp > spatial) rpp = static_cast<int>(spatial);
  const int threads = (vec_per_row * rpp + 31) / 32 * 32;   // whole warps; the surplus threads idle through the loops
  // CTAs per sample: the grid never exceeds the SM count (the CTAs of a sample wait for each other), a CTA gets at
  // least 4 passes of rows
  const int sms = vb_num_sms();
  long long per = n >= sms ? 1 : sms / n;
  const long long max_useful = (spatial + 4LL * rpp - 1) / (4LL * rpp);
  if (per > max_useful) per = max_useful;
  // a sample that fits ONE CTA's shared memory needs no global rendezvous at all (the tiny 5 x 8 level: 10.9 -> ~6 us)
  if (n >= 8 && static_cast<size_t>(spatial) * c * 2 + static_cast<size_t>(rpp) * c * 8 <= 128 * 1024) per = 1;
  if (per < 1) per = 1;
  long long rpc = (spatial + per - 1) / per;
  per = (spatial + rpc - 1) / rpc;
  const size_t part_bytes = static_cast<size_t>(rpp) * c * 2 * sizeof(float);
  const size_t slab_bytes = static_cast<size_t>(rpc) * c * 2;
  const bool cached = part_bytes + slab_bytes <= static_cast<size_t>(GN_DYN_SMEM_MAX);
  const size_t smem = part_bytes + (cached ? slab_bytes : 0);
  p.rpp = rpp; p.threads = threads; p.per = per; p.rpc = rpc; p.cached = cached; p.smem = smem;
  return p;
}

extern "C" int vb200_groupnorm_nhwc(const void* x, const void* weight, const void* bias, void* out,
                                    int64_t n, int64_t spatial, int64_t c, int64_t groups, float eps,
                                    int act, void* workspace, size_t workspace_bytes,
                                    cudaStream_t stream) {
  VB_CHECK_ARG(x && weight && bias && out && n > 0 && spatial > 0 && c > 0 && groups > 0);
  VB_CHECK_ARG(c % 8 == 0 && c % groups == 0);
  VB_CHECK_ARG(c / 8 <= 512 && n <= 65535 && spatial < (1LL << 31) / 4 && groups <= 512);
  VB_CHECK_ARG(act == VB_ACT_NONE || act == VB_ACT_SILU || act == VB_ACT_RELU);
  VB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0);
  const size_t need = vb200_groupnorm_workspace_size(n, groups, c);
  if (!workspace || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 15) != 0) return VB_ERR_WORKSPACE;
  if (n > GN_MAX_N) {
    for (int64_t s0 = 0; s0 < n; s0 += GN_MAX_N) {
      const int64_t ns = n - s0 < GN_MAX_N ? n - s0 : GN_MAX_N;
      const size_t off = static_cast<size_t>(s0) * spatial * c;
      const int r = vb200_groupnorm_nhwc(reinterpret_cast<const bf16*>(x) + off, weight, bias, reinterpret_cast<bf16*>(out) + off, ns,
                                         spatial, c, groups, eps, act, workspace, workspace_bytes, stream);
      if (r != VB_OK) return r;
    }
    return VB_OK;
  }
  GnWs ws;
  char* wsp = reinterpret_cast<char*>(workspace);
  ws.arrived = reinterpret_cast<int*>(wsp);
  ws.readers = ws.arrived + GN_MAX_N;
  ws.sums = reinterpret_cast<float*>(wsp + GN_COUNTER_BYTES);
  GnPlan pl = gn_plan(n, spatial, c);
  if (!pl.cached && n > 1) {
    // The slabs of all n samples do not fit the GPU's shared memory at once (batch-2 UNet levels: 52 MB against 132 x 220 KB):
    // rather than reading x twice, normalise the samples in chunks whose slabs DO fit, one launch per chunk (measured at
    // [2, 40960, 320]: 48 us in one two-pass launch, 2 x 18 us cached). Every chunk uses the same self-zeroing workspace.
    int64_t nc = n;
    while (nc > 1) {
      nc = (nc + 1) / 2;
      if (gn_plan(nc, spatial, c).cached) break;
    }
    if (gn_plan(nc, spatial, c).cached) {
      for (int64_t s0 = 0; s0 < n; s0 += nc) {
        const int64_t ns = n - s0 < nc ? n - s0 : nc;
        const size_t off = static_cast<size_t>(s0) * spatial * c;
        const int r = vb200_groupnorm_nhwc(reinterpret_cast<const bf16*>(x) + off, weight, bias, reinterpret_cast<bf16*>(out) + off, ns,
                                           spatial, c, groups, eps, act, workspace, workspace_bytes, stream);
        if (r != VB_OK) return r;
      }
      return VB_OK;
    }
  }
  const int rpp = pl.rpp, threads = pl.threads;
  const long long per = pl.per, rpc = pl.rpc;
  const bool cached = pl.cached;
  const size_t smem = pl.smem;
  dim3 grid(static_cast<unsigned>(per), static_cast<unsigned>(n));
  const bf16* xp = reinterpret_cast<const bf16*>(x);
  const bf16* wp = reinterpret_cast<const bf16*>(weight);
  const bf16* bp = reinterpret_cast<const bf16*>(bias);
  bf16* op = reinterpret_cast<bf16*>(out);
  const int sp = static_cast<int>(spatial), ci = static_cast<int>(c), gi = static_cast<int>(groups), rc = static_cast<int>(rpc);
#define VB_GN_CASE(A)                                                                                                   \
  return cached ? gn_launch<A, true>(xp, wp, bp, op, ws, sp, ci, gi, rc, rpp, eps, grid, threads, smem, stream)           \
                : gn_launch<A, false>(xp, wp, bp, op, ws, sp, ci, gi, rc, rpp, eps, grid, threads, smem, stream)
  if (act == VB_ACT_SILU) { VB_GN_CASE(VB_ACT_SILU); }
  if (act == VB_ACT_RELU) { VB_GN_CASE(VB_ACT_RELU); }
  VB_GN_CASE(VB_ACT_NONE);
#undef VB_GN_CASE
}
