// vitron_b200 — FocalNet backbone glue kernels (SEEM, SURVEY.md §8 f1; reference
// modules/SEEM/demo_code/xdecoder/backbone/focal.py). All HBM / FP32-pipe bound, NHWC bf16 activations.
//
//   im2col_nchw        stem PatchEmbed Conv2d(3, C, k7, s4, p2) (focal.py:311-338) -> rows for the wgmma GEMM
//   dwconv_gelu<K>     focal_layers[l] = depthwise Conv2d(k, groups=C, bias=False) + GELU (focal.py:80-89,105)
//   colsum / finalize  ctx_global = GELU(mean_hw(ctx)) (focal.py:107), deterministic two-stage reduction
//   focal_modulate     ctx_all = (sum_l ctx_l * gate_l + ctx_global * gate_L) [/ (L+1)] (focal.py:103-111)
//   mul_rows           x_out = q * h(ctx_all) (focal.py:113)
//   layernorm_add      x = shortcut + LN(x) with layerscale folded into the LN affine (focal.py:192-199)
#include "common.cuh"
#include "vitron_b200.h"

namespace vb {

// ------------------------------------------------------------------ helpers
// two fp32 lanes packed in one 64-bit register (sm_90 has no packed FFMA2: fma2 is two FFMAs; the packing costs no
// instructions, the register pair is used in place)
__device__ __forceinline__ unsigned long long pack2(float lo, float hi) {
  unsigned long long r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ float2 unpack2(unsigned long long v) {
  float2 r;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v));
  return r;
}
__device__ __forceinline__ unsigned long long fma2(unsigned long long a, unsigned long long b, unsigned long long c) {
  const float2 x = unpack2(a), y = unpack2(b), z = unpack2(c);
  return pack2(fmaf(x.x, y.x, z.x), fmaf(x.y, y.y, z.y));
}
// packed bf16 pair -> packed fp32 pair (element 0 in the low half)
__device__ __forceinline__ unsigned long long bf2_to_f2(uint32_t w) {
  return pack2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}
struct V8 { unsigned long long p[4]; };
__device__ __forceinline__ V8 unpack8(const uint4 u) {
  V8 r;
  r.p[0] = bf2_to_f2(u.x); r.p[1] = bf2_to_f2(u.y); r.p[2] = bf2_to_f2(u.z); r.p[3] = bf2_to_f2(u.w);
  return r;
}
__device__ __forceinline__ uint4 ldg16(const bf16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// ------------------------------------------------------------------ stem im2col
// out[(n, oy, ox), (c, ky, kx)] = x[n, c, oy*stride - pad + ky, ox*stride - pad + kx] (0 outside the image —
// which also realises the reference's right/bottom zero padding to a multiple of the patch size);
// columns >= c*k*k are zero. One thread = 8 consecutive columns of one row.
__global__ void im2col_nchw_kernel(const void* __restrict__ x, int in_is_fp32, bf16* __restrict__ out, int nb, int c,
                                   int h, int w, int k, int stride, int pad, int ho, int wo, int kpad) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const int vec_per_row = kpad / 8;
  const long long total = static_cast<long long>(nb) * ho * wo * vec_per_row;
  if (idx >= total) return;
  const int v = static_cast<int>(idx % vec_per_row);
  long long r = idx / vec_per_row;
  const int ox = static_cast<int>(r % wo); r /= wo;
  const int oy = static_cast<int>(r % ho);
  const long long n = r / ho;
  const int kk = k * k, kreal = c * kk;
  float f[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = v * 8 + j;
    float val = 0.f;
    if (col < kreal) {
      const int ci = col / kk, rem = col % kk;
      const int iy = oy * stride - pad + rem / k, ix = ox * stride - pad + rem % k;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) {
        const long long off = ((n * c + ci) * h + iy) * static_cast<long long>(w) + ix;
        val = in_is_fp32 ? __ldg(reinterpret_cast<const float*>(x) + off)
                         : __bfloat162float(reinterpret_cast<const bf16*>(x)[off]);
      }
    }
    f[j] = val;
  }
  uint4 o;
  o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]); o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
  reinterpret_cast<uint4*>(out)[idx] = o;
}

// ------------------------------------------------------------------ depthwise conv + GELU
// x: [nb, h, w, ld_in] view (channels [0, c) used), wt: [K*K, c] bf16 (tap-major), out: [nb, h, w, c] contiguous.
// One thread = 8 channels x S consecutive output pixels of one row: per kernel row it loads S+K-1 input
// vectors once (sliding window in registers) and issues K*S*4 FFMA2.
template <int K, int S>
__global__ void __launch_bounds__(128) dwconv_gelu_kernel(const bf16* __restrict__ x, long long ld_in,
                                                          const bf16* __restrict__ wt, bf16* __restrict__ out, int nb,
                                                          int h, int w, int c, int apply_gelu) {
  const int g8 = c / 8;
  const int nxs = (w + S - 1) / S;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;   // the launcher guarantees total < 2^31: 32-bit div / mod
  const unsigned total = static_cast<unsigned>(nb) * h * nxs * g8;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % g8);
  unsigned r = idx / g8;
  const int xs = static_cast<int>(r % nxs); r /= nxs;
  const int y = static_cast<int>(r % h);
  const long long n = r / h;
  const int x0 = xs * S;
  constexpr int R = K / 2;

  unsigned long long acc[S][4];
#pragma unroll
  for (int s = 0; s < S; ++s)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[s][j] = 0ull;

#pragma unroll 1
  for (int ky = 0; ky < K; ++ky) {
    const int iy = y + ky - R;
    if (iy < 0 || iy >= h) continue;
    const bf16* rowp = x + ((n * h + iy) * static_cast<long long>(w)) * ld_in + cg * 8;
    V8 v[S + K - 1];
#pragma unroll
    for (int i = 0; i < S + K - 1; ++i) {
      const int ix = x0 - R + i;
      uint4 u = make_uint4(0u, 0u, 0u, 0u);
      if (ix >= 0 && ix < w) u = ldg16(rowp + static_cast<long long>(ix) * ld_in);
      v[i] = unpack8(u);
    }
    const bf16* wrow = wt + static_cast<long long>(ky * K) * c + cg * 8;
#pragma unroll
    for (int kx = 0; kx < K; ++kx) {
      const V8 wv = unpack8(ldg16(wrow + static_cast<long long>(kx) * c));
#pragma unroll
      for (int s = 0; s < S; ++s)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[s][j] = fma2(v[s + kx].p[j], wv.p[j], acc[s][j]);
    }
  }
  bf16* orow = out + ((n * h + y) * static_cast<long long>(w)) * c + cg * 8;
#pragma unroll
  for (int s = 0; s < S; ++s) {
    if (x0 + s >= w) break;
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = unpack2(acc[s][j]);
      f[2 * j] = apply_gelu ? gelu_erf_fast(t.x) : t.x;
      f[2 * j + 1] = apply_gelu ? gelu_erf_fast(t.y) : t.y;
    }
    uint4 o;
    o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]); o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
    *reinterpret_cast<uint4*>(orow + static_cast<long long>(x0 + s) * c) = o;
  }
}

// v2 (default): one thread = ONE bf16 channel pair x S consecutive output pixels of a row. A warp's 32 lanes
// read 128 contiguous bytes of a pixel (full sectors); every input word is converted to a packed fp32 pair once
// (2 ALU ops) and feeds up to K FFMA2, the K weights of the kernel row sit in registers: (S+K-1)*2 + K*2 ALU ops
// per S*K FFMA2 (S = 32, K = 9: 98 vs 288) instead of the 1 : 1 of the 8-channel variant above.
template <int K, int S>
__global__ void __launch_bounds__(128) dwconv_gelu_pair_kernel(const bf16* __restrict__ x, long long ld_in,
                                                               const bf16* __restrict__ wt, bf16* __restrict__ out,
                                                               int nb, int h, int w, int c, int apply_gelu) {
  const int c2n = c / 2;
  const int nxs = (w + S - 1) / S;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;   // the launcher guarantees total < 2^31: 32-bit div / mod
  const unsigned total = static_cast<unsigned>(nb) * h * nxs * c2n;
  if (idx >= total) return;
  const int cp = static_cast<int>(idx % c2n);
  unsigned r = idx / c2n;
  const int xs = static_cast<int>(r % nxs); r /= nxs;
  const int y = static_cast<int>(r % h);
  const long long n = r / h;
  const int x0 = xs * S;
  constexpr int R = K / 2;
  const int ldw = static_cast<int>(ld_in / 2);  // pixel stride in 32-bit words (32-bit: one IMAD.WIDE per address)
  const uint32_t* wt32 = reinterpret_cast<const uint32_t*>(wt) + cp;
  // strips whose whole input window lies inside the row take the predicate-free path
  const bool interior = (x0 - R >= 0) && (x0 + S - 1 + R < w);

  unsigned long long acc[S];
#pragma unroll
  for (int s = 0; s < S; ++s) acc[s] = 0ull;

#pragma unroll 1
  for (int ky = 0; ky < K; ++ky) {
    const int iy = y + ky - R;
    if (iy < 0 || iy >= h) continue;
    // first word of the window (may lie left of the row start for edge strips: only dereferenced when in range)
    const uint32_t* p0 = reinterpret_cast<const uint32_t*>(x + ((n * h + iy) * static_cast<long long>(w)) * ld_in) + cp +
                         static_cast<long long>(x0 - R) * ldw;
    uint32_t pk[S + K - 1];
    if (interior) {
#pragma unroll
      for (int i = 0; i < S + K - 1; ++i) pk[i] = __ldg(p0 + i * ldw);
    } else {
#pragma unroll
      for (int i = 0; i < S + K - 1; ++i) {
        const int ix = x0 - R + i;
        pk[i] = (ix >= 0 && ix < w) ? __ldg(p0 + i * ldw) : 0u;
      }
    }
    unsigned long long wv[K];
#pragma unroll
    for (int kx = 0; kx < K; ++kx) wv[kx] = bf2_to_f2(__ldg(wt32 + (ky * K + kx) * c2n));
#pragma unroll
    for (int i = 0; i < S + K - 1; ++i) {
      const unsigned long long v = bf2_to_f2(pk[i]);
#pragma unroll
      for (int kx = 0; kx < K; ++kx) {
        const int s = i - kx;
        if (s >= 0 && s < S) acc[s] = fma2(v, wv[kx], acc[s]);
      }
    }
  }
  uint32_t* orow = reinterpret_cast<uint32_t*>(out + ((n * h + y) * static_cast<long long>(w)) * c) + cp;
#pragma unroll
  for (int s = 0; s < S; ++s) {
    if (x0 + s >= w) break;
    float2 t = unpack2(acc[s]);
    if (apply_gelu) { t.x = gelu_erf_fast(t.x); t.y = gelu_erf_fast(t.y); }
    orow[static_cast<long long>(x0 + s) * c2n] = pack_bf16(t.x, t.y);
  }
}

// ------------------------------------------------------------------ column sums (global context)
// x [nb, t, c] contiguous bf16 -> partial [nb, nchunks, c] fp32 (sum over the chunk's rows). grid (nchunks, nb).
__global__ void __launch_bounds__(256) colsum_partial_kernel(const bf16* __restrict__ x, float* __restrict__ partial,
                                                             long long t, int c, int rows_per_chunk) {
  extern __shared__ float sred[];  // [nrl][c]
  const int g8 = c / 8;
  const int nrl = 256 / g8;  // row lanes (>= 1 because c <= 2048)
  const int cg = threadIdx.x % g8, rl = threadIdx.x / g8;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_chunk;
  const long long r1 = min(r0 + rows_per_chunk, t);
  float s[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = 0.f;
  if (rl < nrl) {
    const bf16* base = x + (static_cast<long long>(blockIdx.y) * t) * c + cg * 8;
    auto add8 = [&](const uint4 u) {
      float2 f;
      f = unpack_bf16(u.x); s[0] += f.x; s[1] += f.y;
      f = unpack_bf16(u.y); s[2] += f.x; s[3] += f.y;
      f = unpack_bf16(u.z); s[4] += f.x; s[5] += f.y;
      f = unpack_bf16(u.w); s[6] += f.x; s[7] += f.y;
    };
    long long r = r0 + rl;
    for (; r + 3ll * nrl < r1; r += 4ll * nrl) {  // four independent 16-byte loads in flight
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = ldg16(base + (r + static_cast<long long>(k) * nrl) * c);
#pragma unroll
      for (int k = 0; k < 4; ++k) add8(u[k]);
    }
    for (; r < r1; r += nrl) add8(ldg16(base + r * c));
#pragma unroll
    for (int j = 0; j < 8; ++j) sred[rl * c + cg * 8 + j] = s[j];
  }
  __syncthreads();
  float* dst = partial + (static_cast<long long>(blockIdx.y) * gridDim.x + blockIdx.x) * c;
  for (int ch = threadIdx.x; ch < c; ch += 256) {
    float a = 0.f;
    for (int l = 0; l < nrl; ++l) a += sred[l * c + ch];  // fixed order: deterministic
    dst[ch] = a;
  }
}

// glob[b, ch] = act(sum_chunks partial / t). grid (c / 32, nb), block (32 channels, 32 chunk lanes): every lane adds
// its strided share of the chunks, then a fixed-order shared-memory tree -> deterministic, and ~nchunks/32 dependent
// loads per thread instead of nchunks.
__global__ void __launch_bounds__(1024) colmean_finalize_kernel(const float* __restrict__ partial, float* __restrict__ glob,
                                                                int nchunks, int c, float inv_t, int apply_gelu) {
  __shared__ float red[32][33];
  const int ch = blockIdx.x * 32 + threadIdx.x;
  const int b = blockIdx.y;
  float a = 0.f;
  if (ch < c) {
    const float* p = partial + static_cast<long long>(b) * nchunks * c + ch;
    for (int k = threadIdx.y; k < nchunks; k += 32) a += p[static_cast<long long>(k) * c];
  }
  red[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && ch < c) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) t += red[k][threadIdx.x];
    t *= inv_t;
    glob[b * c + ch] = apply_gelu ? gelu_erf(t) : t;
  }
}

// ------------------------------------------------------------------ focal modulation
struct FocalCtx {
  const bf16* ctx[VB_FOCAL_MAX_LEVELS];
};
// out[pix, ch] = scale * (sum_l ctx_l[pix, ch] * gates[pix, l] + glob[b, ch] * gates[pix, nlev])
__global__ void focal_modulate_kernel(FocalCtx cx, int nlev, const bf16* __restrict__ gates, long long ld_g,
                                      const float* __restrict__ glob, bf16* __restrict__ out, long long t, int c, int nb,
                                      float scale) {
  const int g8 = c / 8;
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long total = static_cast<long long>(nb) * t * g8;
  if (idx >= total) return;
  const int cg = static_cast<int>(idx % g8);
  const long long pix = idx / g8;
  const long long b = pix / t;
  const bf16* gp = gates + pix * ld_g;
  float a[8];
  {
    const float gl = __bfloat162float(gp[nlev]);
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(glob + b * c + cg * 8));
    const float4 g1 = __ldg(reinterpret_cast<const float4*>(glob + b * c + cg * 8 + 4));
    a[0] = g0.x * gl; a[1] = g0.y * gl; a[2] = g0.z * gl; a[3] = g0.w * gl;
    a[4] = g1.x * gl; a[5] = g1.y * gl; a[6] = g1.z * gl; a[7] = g1.w * gl;
  }
  for (int l = 0; l < nlev; ++l) {
    const float gl = __bfloat162float(gp[l]);
    const uint4 u = ldg16(cx.ctx[l] + pix * c + cg * 8);
    float2 f;
    f = unpack_bf16(u.x); a[0] = fmaf(f.x, gl, a[0]); a[1] = fmaf(f.y, gl, a[1]);
    f = unpack_bf16(u.y); a[2] = fmaf(f.x, gl, a[2]); a[3] = fmaf(f.y, gl, a[3]);
    f = unpack_bf16(u.z); a[4] = fmaf(f.x, gl, a[4]); a[5] = fmaf(f.y, gl, a[5]);
    f = unpack_bf16(u.w); a[6] = fmaf(f.x, gl, a[6]); a[7] = fmaf(f.y, gl, a[7]);
  }
  uint4 o;
  o.x = pack_bf16(a[0] * scale, a[1] * scale); o.y = pack_bf16(a[2] * scale, a[3] * scale);
  o.z = pack_bf16(a[4] * scale, a[5] * scale); o.w = pack_bf16(a[6] * scale, a[7] * scale);
  *reinterpret_cast<uint4*>(out + pix * c + cg * 8) = o;
}

// out[row, :] = a[row, :] (row stride ld_a) * b[row, :] (row stride ld_b), c columns
__global__ void mul_rows_kernel(const bf16* __restrict__ a, long long ld_a, const bf16* __restrict__ b, long long ld_b,
                                bf16* __restrict__ out, long long rows, int c) {
  const int g8 = c / 8;
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= rows * g8) return;
  const int cg = static_cast<int>(idx % g8);
  const long long row = idx / g8;
  const uint4 ua = ldg16(a + row * ld_a + cg * 8), ub = ldg16(b + row * ld_b + cg * 8);
  const float2 a0 = unpack_bf16(ua.x), a1 = unpack_bf16(ua.y), a2 = unpack_bf16(ua.z), a3 = unpack_bf16(ua.w);
  const float2 b0 = unpack_bf16(ub.x), b1 = unpack_bf16(ub.y), b2 = unpack_bf16(ub.z), b3 = unpack_bf16(ub.w);
  uint4 o;
  o.x = pack_bf16(a0.x * b0.x, a0.y * b0.y); o.y = pack_bf16(a1.x * b1.x, a1.y * b1.y);
  o.z = pack_bf16(a2.x * b2.x, a2.y * b2.y); o.w = pack_bf16(a3.x * b3.x, a3.y * b3.y);
  *reinterpret_cast<uint4*>(out + row * c + cg * 8) = o;
}

// ------------------------------------------------------------------ LayerNorm (+ residual)
// out[row] = res[row] + LN(x[row]) * w + b ; one warp per ROWS rows, rows held in registers (d <= 256 * MAXV, d % 8 == 0),
// statistics in fp32, two passes over the registers (mean, then centred variance). Every global load of the warp's
// rows (x AND the residual) is issued before the first reduction, so a warp has ROWS * MAXV * 2 loads in flight.
template <int MAXV, int ROWS>
__global__ void __launch_bounds__(256) layernorm_add_kernel(const bf16* __restrict__ x, long long ldx,
                                                            const bf16* __restrict__ w, const bf16* __restrict__ b,
                                                            const bf16* __restrict__ res, long long ldr,
                                                            bf16* __restrict__ out, long long ldo, long long rows, int d,
                                                            float eps) {
  const long long row0 = (blockIdx.x * 8ll + (threadIdx.x >> 5)) * ROWS;
  if (row0 >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nvec = d / 8;
  uint4 u[ROWS][MAXV], ur[ROWS][MAXV];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const bool live = row0 + r < rows;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int v = lane + 32 * i;
      u[r][i] = make_uint4(0u, 0u, 0u, 0u);
      ur[r][i] = make_uint4(0u, 0u, 0u, 0u);
      if (live && v < nvec) {
        u[r][i] = ldg16(x + (row0 + r) * ldx + v * 8);
        if (res) ur[r][i] = ldg16(res + (row0 + r) * ldr + v * 8);
      }
    }
  }
  float mean[ROWS], rstd[ROWS];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      float2 f;
      f = unpack_bf16(u[r][i].x); sum += f.x + f.y;
      f = unpack_bf16(u[r][i].y); sum += f.x + f.y;
      f = unpack_bf16(u[r][i].z); sum += f.x + f.y;
      f = unpack_bf16(u[r][i].w); sum += f.x + f.y;
    }
    mean[r] = warp_sum(sum) / static_cast<float>(d);
  }
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    float sq = 0.f;
    const float m = mean[r];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      if (lane + 32 * i < nvec) {
        float2 f;
        f = unpack_bf16(u[r][i].x); sq += (f.x - m) * (f.x - m) + (f.y - m) * (f.y - m);
        f = unpack_bf16(u[r][i].y); sq += (f.x - m) * (f.x - m) + (f.y - m) * (f.y - m);
        f = unpack_bf16(u[r][i].z); sq += (f.x - m) * (f.x - m) + (f.y - m) * (f.y - m);
        f = unpack_bf16(u[r][i].w); sq += (f.x - m) * (f.x - m) + (f.y - m) * (f.y - m);
      }
    }
    rstd[r] = rsqrtf(warp_sum(sq) / static_cast<float>(d) + eps);
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = lane + 32 * i;
    if (v >= nvec) continue;
    const uint4 uw = ldg16(w + v * 8);
    uint4 ub = make_uint4(0u, 0u, 0u, 0u);
    if (b) ub = ldg16(b + v * 8);
    const uint32_t ws[4] = {uw.x, uw.y, uw.z, uw.w};
    const uint32_t bs[4] = {ub.x, ub.y, ub.z, ub.w};
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      if (row0 + r >= rows) break;
      const uint32_t xs[4] = {u[r][i].x, u[r][i].y, u[r][i].z, u[r][i].w};
      const uint32_t rs[4] = {ur[r][i].x, ur[r][i].y, ur[r][i].z, ur[r][i].w};
      uint32_t os[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 fx = unpack_bf16(xs[j]), fw = unpack_bf16(ws[j]), fb = unpack_bf16(bs[j]), fr = unpack_bf16(rs[j]);
        os[j] = pack_bf16(fr.x + (fx.x - mean[r]) * rstd[r] * fw.x + fb.x, fr.y + (fx.y - mean[r]) * rstd[r] * fw.y + fb.y);
      }
      *reinterpret_cast<uint4*>(out + (row0 + r) * ldo + v * 8) = make_uint4(os[0], os[1], os[2], os[3]);
    }
  }
}

}  // namespace vb

using namespace vb;

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int vb200_im2col_nchw(const void* pixels, int in_is_fp32, void* out, int64_t nb, int64_t c, int64_t h,
                                 int64_t w, int64_t k, int64_t stride, int64_t pad, int64_t ho, int64_t wo,
                                 int64_t kpad, cudaStream_t stream) {
  VB_CHECK_ARG(pixels && out && nb > 0 && c > 0 && h > 0 && w > 0 && k > 0 && stride > 0 && pad >= 0);
  VB_CHECK_ARG(ho > 0 && wo > 0 && kpad % 8 == 0 && kpad >= c * k * k && aligned16(out));
  const long long total = nb * ho * wo * (kpad / 8);
  im2col_nchw_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      pixels, in_is_fp32, reinterpret_cast<bf16*>(out), (int)nb, (int)c, (int)h, (int)w, (int)k, (int)stride, (int)pad,
      (int)ho, (int)wo, (int)kpad);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

template <int K, int S>
static int launch_dwconv(const void* x, int64_t ld_in, const void* wt, void* out, int64_t nb, int64_t h, int64_t w,
                         int64_t c, int act, cudaStream_t stream) {
  const long long total = nb * h * ((w + S - 1) / S) * (c / 8);
  dwconv_gelu_kernel<K, S><<<static_cast<unsigned>((total + 127) / 128), 128, 0, stream>>>(
      reinterpret_cast<const bf16*>(x), ld_in, reinterpret_cast<const bf16*>(wt), reinterpret_cast<bf16*>(out), (int)nb,
      (int)h, (int)w, (int)c, act);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

static int g_dwconv_impl = 0;  // 0 = automatic, 1 = 8-channel kernel, 2 / 3 = channel-pair kernel with 16 / 32-pixel strips
extern "C" int vb200_set_dwconv_impl(int impl) {
  const int prev = g_dwconv_impl;
  if (impl >= 0 && impl <= 3) g_dwconv_impl = impl;
  return prev;
}

template <int K>
static int launch_dwconv_pair(const void* x, int64_t ld_in, const void* wt, void* out, int64_t nb, int64_t h, int64_t w,
                              int64_t c, int act, cudaStream_t stream) {
  const long long c2n = c / 2;
  const long long t32 = nb * h * ((w + 31) / 32) * c2n;
  const bf16* xp = reinterpret_cast<const bf16*>(x);
  const bf16* wp = reinterpret_cast<const bf16*>(wt);
  bf16* op = reinterpret_cast<bf16*>(out);
  // 32-pixel strips re-read the fewest halo columns but need ~250 registers; they pay off only when there are
  // enough strips to fill the machine several times over and the kernel is small enough not to spill
  const bool wide = g_dwconv_impl == 3;  // opt-in only: the 16-pixel strips are the default at every k
  if (wide) {
    dwconv_gelu_pair_kernel<K, 32><<<static_cast<unsigned>((t32 + 127) / 128), 128, 0, stream>>>(xp, ld_in, wp, op, (int)nb,
                                                                                                  (int)h, (int)w, (int)c, act);
  } else {
    const long long t16 = nb * h * ((w + 15) / 16) * c2n;
    dwconv_gelu_pair_kernel<K, 16><<<static_cast<unsigned>((t16 + 127) / 128), 128, 0, stream>>>(xp, ld_in, wp, op, (int)nb,
                                                                                                  (int)h, (int)w, (int)c, act);
  }
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_dwconv_nhwc(const void* x, int64_t ld_in, const void* wt, void* out, int64_t nb, int64_t h,
                                 int64_t w, int64_t c, int64_t k, int act, cudaStream_t stream) {
  VB_CHECK_ARG(x && wt && out && nb > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0 && ld_in % 8 == 0 && ld_in >= c);
  VB_CHECK_ARG(aligned16(x) && aligned16(wt) && aligned16(out));
  VB_CHECK_ARG(act == VB_ACT_NONE || act == VB_ACT_GELU);
  VB_CHECK_ARG(nb * h * ((w + 3) / 4) * (c / 2) < (1ll << 31) - 256);  // thread indices of every variant fit 32 bits
  VB_CHECK_ARG(nb * h * w * ld_in < (1ll << 33));
  const int g = act == VB_ACT_GELU ? 1 : 0;
  // automatic: k = 3 / 5 are load-bound -> the 16-byte loads of the 8-channel kernel; k >= 7 is instruction-bound -> the
  // channel-pair kernel (fewer conversions per FMA)
  if (g_dwconv_impl >= 2 || (g_dwconv_impl == 0 && k >= 7)) {
    switch (k) {
      case 3: return launch_dwconv_pair<3>(x, ld_in, wt, out, nb, h, w, c, g, stream);
      case 5: return launch_dwconv_pair<5>(x, ld_in, wt, out, nb, h, w, c, g, stream);
      case 7: return launch_dwconv_pair<7>(x, ld_in, wt, out, nb, h, w, c, g, stream);
      case 9: return launch_dwconv_pair<9>(x, ld_in, wt, out, nb, h, w, c, g, stream);
      case 11: return launch_dwconv_pair<11>(x, ld_in, wt, out, nb, h, w, c, g, stream);
      default: return VB_ERR_UNSUPPORTED;
    }
  }
  switch (k) {
    case 3: return launch_dwconv<3, 8>(x, ld_in, wt, out, nb, h, w, c, g, stream);
    case 5: return launch_dwconv<5, 8>(x, ld_in, wt, out, nb, h, w, c, g, stream);
    case 7: return launch_dwconv<7, 4>(x, ld_in, wt, out, nb, h, w, c, g, stream);
    case 9: return launch_dwconv<9, 4>(x, ld_in, wt, out, nb, h, w, c, g, stream);
    case 11: return launch_dwconv<11, 4>(x, ld_in, wt, out, nb, h, w, c, g, stream);
    default: return VB_ERR_UNSUPPORTED;
  }
}

static inline int colsum_chunks(int64_t t) {
  // enough CTAs to cover the machine twice (the reduction is latency bound per thread), >= 16 rows per chunk
  int64_t n = (t + 15) / 16;
  const int64_t cap = 2 * static_cast<int64_t>(vb_num_sms());
  return static_cast<int>(n < 1 ? 1 : (n > cap ? cap : n));
}

extern "C" size_t vb200_colmean_workspace_size(int64_t nb, int64_t t, int64_t c) {
  return static_cast<size_t>(nb) * colsum_chunks(t) * c * sizeof(float);
}

extern "C" int vb200_colmean(const void* x, float* out, int64_t nb, int64_t t, int64_t c, int act, void* workspace,
                             size_t workspace_bytes, cudaStream_t stream) {
  VB_CHECK_ARG(x && out && nb > 0 && t > 0 && c > 0 && c % 8 == 0 && c <= 2048 && aligned16(x));
  VB_CHECK_ARG(act == VB_ACT_NONE || act == VB_ACT_GELU);
  const int nchunks = colsum_chunks(t);
  if (workspace == nullptr || workspace_bytes < vb200_colmean_workspace_size(nb, t, c)) return VB_ERR_WORKSPACE;
  const int rows_per_chunk = static_cast<int>((t + nchunks - 1) / nchunks);
  const int nrl = 256 / static_cast<int>(c / 8);
  const size_t smem = static_cast<size_t>(nrl) * c * sizeof(float);
  colsum_partial_kernel<<<dim3(nchunks, (unsigned)nb), 256, smem, stream>>>(reinterpret_cast<const bf16*>(x),
                                                                           reinterpret_cast<float*>(workspace), t, (int)c,
                                                                           rows_per_chunk);
  VB_LAUNCH_CHECK();
  colmean_finalize_kernel<<<dim3(static_cast<unsigned>((c + 31) / 32), (unsigned)nb), dim3(32, 32), 0, stream>>>(
      reinterpret_cast<const float*>(workspace), out, nchunks, (int)c, 1.0f / static_cast<float>(t), act == VB_ACT_GELU ? 1 : 0);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_focal_modulate(const void* const* ctx_levels, int64_t nlev, const void* gates, int64_t ld_g,
                                    const float* glob, void* out, int64_t nb, int64_t t, int64_t c, float scale,
                                    cudaStream_t stream) {
  VB_CHECK_ARG(ctx_levels && gates && glob && out && nlev > 0 && nlev <= VB_FOCAL_MAX_LEVELS);
  VB_CHECK_ARG(nb > 0 && t > 0 && c > 0 && c % 8 == 0 && aligned16(out) && aligned16(glob));
  FocalCtx cx;
  for (int l = 0; l < VB_FOCAL_MAX_LEVELS; ++l) {
    cx.ctx[l] = l < nlev ? reinterpret_cast<const bf16*>(ctx_levels[l]) : nullptr;
    if (l < nlev) VB_CHECK_ARG(ctx_levels[l] != nullptr && aligned16(ctx_levels[l]));
  }
  const long long total = nb * t * (c / 8);
  focal_modulate_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      cx, (int)nlev, reinterpret_cast<const bf16*>(gates), ld_g, glob, reinterpret_cast<bf16*>(out), t, (int)c, (int)nb,
      scale);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_mul_rows(const void* a, int64_t ld_a, const void* b, int64_t ld_b, void* out, int64_t rows,
                              int64_t c, cudaStream_t stream) {
  VB_CHECK_ARG(a && b && out && rows >= 0 && c > 0 && c % 8 == 0 && ld_a % 8 == 0 && ld_b % 8 == 0);
  VB_CHECK_ARG(aligned16(a) && aligned16(b) && aligned16(out));
  if (rows == 0) return VB_OK;
  const long long total = rows * (c / 8);
  mul_rows_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const bf16*>(a), ld_a, reinterpret_cast<const bf16*>(b), ld_b, reinterpret_cast<bf16*>(out), rows,
      (int)c);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_layernorm_add(const void* x, int64_t ldx, const void* weight, const void* bias, const void* residual,
                                   int64_t ldr, void* out, int64_t ldo, int64_t rows, int64_t d, float eps,
                                   cudaStream_t stream) {
  VB_CHECK_ARG(x && weight && out && rows >= 0 && d > 0 && d % 8 == 0 && d <= 2048);
  VB_CHECK_ARG(ldx % 8 == 0 && ldo % 8 == 0 && (residual == nullptr || ldr % 8 == 0));
  VB_CHECK_ARG(aligned16(x) && aligned16(weight) && aligned16(out) && aligned16(bias) && aligned16(residual));
  if (rows == 0) return VB_OK;
  const bf16* xp = reinterpret_cast<const bf16*>(x);
  const bf16* wp = reinterpret_cast<const bf16*>(weight);
  const bf16* bp = reinterpret_cast<const bf16*>(bias);
  const bf16* rp = reinterpret_cast<const bf16*>(residual);
  bf16* op = reinterpret_cast<bf16*>(out);
  auto grid = [&](int rows_per_warp) { return static_cast<unsigned>((rows + 8ll * rows_per_warp - 1) / (8ll * rows_per_warp)); };
  if (d <= 256) layernorm_add_kernel<1, 4><<<grid(4), 256, 0, stream>>>(xp, ldx, wp, bp, rp, ldr, op, ldo, rows, (int)d, eps);
  else if (d <= 512) layernorm_add_kernel<2, 4><<<grid(4), 256, 0, stream>>>(xp, ldx, wp, bp, rp, ldr, op, ldo, rows, (int)d, eps);
  else if (d <= 1024) layernorm_add_kernel<4, 2><<<grid(2), 256, 0, stream>>>(xp, ldx, wp, bp, rp, ldr, op, ldo, rows, (int)d, eps);
  else layernorm_add_kernel<8, 1><<<grid(1), 256, 0, stream>>>(xp, ldx, wp, bp, rp, ldr, op, ldo, rows, (int)d, eps);
  VB_LAUNCH_CHECK();
  return VB_OK;
}
