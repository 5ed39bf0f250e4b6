// vitron_b200 — vision / diffusion glue kernels (all HBM-bound, coalesced, no data reuse):
// patchify + ViT embedding/pre-LN, nearest upsample, adds, CFG combine, region mask pooling,
// SEEM attention-mask head, and a direct convolution for the two odd-shaped UNet layers.
#include "common.cuh"
#include "vitron_b200.h"

namespace vb {

// pixels [nb, c, h, w] (fp32 or bf16) -> rows [nb*gh*gw, kpad], k = (ch*patch + py)*patch + px
// (the flattening order of Conv2d weight [out, c, p, p]); columns >= c*p*p are zero.
template <typename T>
__global__ void patchify_kernel(const T* __restrict__ px, bf16* __restrict__ out, int c, int h, int w,
                                int patch, int kpad, long long total) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int k = static_cast<int>(idx % kpad);
  const long long row = idx / kpad;
  const int gw = w / patch, gh = h / patch;
  const int gx = static_cast<int>(row % gw);
  const int gy = static_cast<int>((row / gw) % gh);
  const long long n = row / (static_cast<long long>(gw) * gh);
  float v = 0.f;
  if (k < c * patch * patch) {
    const int pxx = k % patch, pyy = (k / patch) % patch, ch = k / (patch * patch);
    v = static_cast<float>(px[((n * c + ch) * h + gy * patch + pyy) * w + gx * patch + pxx]);
  }
  out[idx] = __float2bfloat16(v);
}

// hidden[b, 0] = LN(cls + pos[0]); hidden[b, 1+p] = LN(patch_out[b*np + p] + pos[1+p])
__global__ void __launch_bounds__(128)
vit_embed_ln_kernel(const bf16* __restrict__ patch_out, const bf16* __restrict__ cls, const bf16* __restrict__ pos,
                    const bf16* __restrict__ w, const bf16* __restrict__ b, bf16* __restrict__ out, int npatch,
                    int d, float eps) {
  __shared__ float red[4];
  const long long row = blockIdx.x;
  const int tok = static_cast<int>(row % (npatch + 1));
  const long long img = row / (npatch + 1);
  const bf16* src = tok == 0 ? cls : patch_out + (img * npatch + tok - 1) * d;
  const bf16* pr = pos + static_cast<long long>(tok) * d;
  float v[16];  // d <= 2048 -> 16 per thread at 128 threads (ViT-H/14: 1280)
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int c = threadIdx.x + i * 128;
    v[i] = c < d ? __bfloat162float(__float2bfloat16(__bfloat162float(src[c]) + __bfloat162float(pr[c]))) : 0.f;
    s += v[i];
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  const float mean = (red[0] + red[1] + red[2] + red[3]) / d;
  __syncthreads();
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int c = threadIdx.x + i * 128;
    if (c < d) { const float t = v[i] - mean; q += t * t; }
  }
  q = warp_sum(q);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = q;
  __syncthreads();
  const float rstd = rsqrtf((red[0] + red[1] + red[2] + red[3]) / d + eps);
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int c = threadIdx.x + i * 128;
    if (c < d)
      out[row * d + c] = __float2bfloat16((v[i] - mean) * rstd * __bfloat162float(w[c]) + __bfloat162float(b[c]));
  }
}

__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int h, int w, int cv,
                                  long long total) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int c = static_cast<int>(idx % cv);
  long long r = idx / cv;
  const int ox = static_cast<int>(r % (2 * w)); r /= (2 * w);
  const int oy = static_cast<int>(r % (2 * h));
  const long long n = r / (2 * h);
  out[idx] = x[((n * h + oy / 2) * w + ox / 2) * cv + c];
}

__global__ void add_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ out,
                           long long nvec, long long period_vec) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= nvec) return;
  const uint4 x = a[idx], y = b[period_vec > 0 ? idx % period_vec : idx];
  const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float2 f = unpack_bf16(xs[j]), g = unpack_bf16(ys[j]);
    o[j] = pack_bf16(f.x + g.x, f.y + g.y);
  }
  out[idx] = make_uint4(o[0], o[1], o[2], o[3]);
}

__global__ void add_rowgroup_kernel(const uint4* __restrict__ x, const uint4* __restrict__ table, uint4* __restrict__ out,
                                    long long nvec, int dv, long long group_rows, long long period) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= nvec) return;
  const long long row = idx / dv;
  const int c = static_cast<int>(idx % dv);
  const uint4 a = x[idx], b = table[((row / group_rows) % period) * dv + c];
  const uint32_t xs[4] = {a.x, a.y, a.z, a.w}, ys[4] = {b.x, b.y, b.z, b.w};
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float2 f = unpack_bf16(xs[j]), g = unpack_bf16(ys[j]);
    o[j] = pack_bf16(f.x + g.x, f.y + g.y);
  }
  out[idx] = make_uint4(o[0], o[1], o[2], o[3]);
}

__global__ void cfg_kernel(const float* __restrict__ y, const float* __restrict__ u, float* __restrict__ out,
                           float s, long long n) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx < n) out[idx] = u[idx] + s * (y[idx] - u[idx]);
}

// bilinear (align_corners=False, no antialias) sample of a box indicator on an S x S canvas at the
// centre of cell (gy, gx) of a g x g grid; mask[int(x1):int(x2), int(y1):int(y2)] = 1 (x -> rows).
__device__ __forceinline__ float box_bilinear(float x1, float y1, float x2, float y2, int S, int g, int gy, int gx) {
  const int r0 = max(0, min(S, static_cast<int>(x1))), r1 = max(0, min(S, static_cast<int>(x2)));
  const int c0 = max(0, min(S, static_cast<int>(y1))), c1 = max(0, min(S, static_cast<int>(y2)));
  const float scale = static_cast<float>(S) / g;
  float sy = (gy + 0.5f) * scale - 0.5f, sx = (gx + 0.5f) * scale - 0.5f;
  sy = fmaxf(sy, 0.f); sx = fmaxf(sx, 0.f);
  const int y0 = min(static_cast<int>(sy), S - 1), x0 = min(static_cast<int>(sx), S - 1);
  const int y1i = min(y0 + 1, S - 1), x1i = min(x0 + 1, S - 1);
  const float ly = sy - y0, lx = sx - x0;
  auto in = [&](int r, int c) { return (r >= r0 && r < r1 && c >= c0 && c < c1) ? 1.f : 0.f; };
  return (1 - ly) * ((1 - lx) * in(y0, x0) + lx * in(y0, x1i)) + ly * ((1 - lx) * in(y1i, x0) + lx * in(y1i, x1i));
}

__global__ void region_pool_kernel(const bf16* __restrict__ feats, const float* __restrict__ boxes,
                                   bf16* __restrict__ out, int g, int c, int S) {
  // one CTA per (batch, 256-channel slab); cell weights computed once into smem
  extern __shared__ float wts[];  // [g*g]
  const int b = blockIdx.y;
  const float* bx = boxes + b * 4;
  float local = 0.f;
  for (int i = threadIdx.x; i < g * g; i += blockDim.x) {
    const float m = box_bilinear(bx[0], bx[1], bx[2], bx[3], S, g, i / g, i % g) > 0.f ? 1.f : 0.f;
    wts[i] = m;
    local += m;
  }
  __shared__ float red[32];
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  float cnt = 0.f;
  for (int i = 0; i < (blockDim.x >> 5); ++i) cnt += red[i];
  const float inv = 1.f / (cnt + 1e-8f);
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  const bf16* f = feats + static_cast<long long>(b) * g * g * c + ch;
  float acc = 0.f;
  for (int i = 0; i < g * g; ++i)
    if (wts[i] != 0.f) acc += __bfloat162float(f[static_cast<long long>(i) * c]) * inv;
  out[static_cast<long long>(b) * c + ch] = __float2bfloat16(acc);
}

// SEEM: logits [Q, H, W] fp32 -> mask [Q, h2*w2] uint8 (1 = masked out) = (sigmoid(bilinear) < 0.5),
// then rows that are entirely masked are cleared. One CTA per query.
__global__ void __launch_bounds__(256)
seem_mask_kernel(const float* __restrict__ logits, uint8_t* __restrict__ out, int H, int W, int h2, int w2) {
  __shared__ int any_open;
  const int qi = blockIdx.x;
  const float* src = logits + static_cast<long long>(qi) * H * W;
  uint8_t* dst = out + static_cast<long long>(qi) * h2 * w2;
  if (threadIdx.x == 0) any_open = 0;
  __syncthreads();
  const float sh = static_cast<float>(H) / h2, sw = static_cast<float>(W) / w2;
  int open_local = 0;
  for (int i = threadIdx.x; i < h2 * w2; i += blockDim.x) {
    const int oy = i / w2, ox = i % w2;
    float sy = fmaxf((oy + 0.5f) * sh - 0.5f, 0.f), sx = fmaxf((ox + 0.5f) * sw - 0.5f, 0.f);
    const int y0 = min(static_cast<int>(sy), H - 1), x0 = min(static_cast<int>(sx), W - 1);
    const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float ly = sy - y0, lx = sx - x0;
    const float v = (1 - ly) * ((1 - lx) * src[y0 * W + x0] + lx * src[y0 * W + x1]) +
                    ly * ((1 - lx) * src[y1 * W + x0] + lx * src[y1 * W + x1]);
    // sigmoid(v) < 0.5  <=>  v < 0
    const uint8_t masked = v < 0.f ? 1 : 0;
    dst[i] = masked;
    open_local |= !masked;
  }
  if (open_local) atomicOr(&any_open, 1);
  __syncthreads();
  if (!any_open)
    for (int i = threadIdx.x; i < h2 * w2; i += blockDim.x) dst[i] = 0;
}

// Bilinear (align_corners=False, no antialias = F.interpolate) resize of NHWC bf16 images; one thread per (output pixel,
// 8 channels). SEEM: the next layer's attention-mask logits are bilinear(mask_embed . mask_features) — bilinear resizing is
// linear in the pixel axis, so resizing mask_features ONCE per level and multiplying the 101 mask embeddings with the small
// map gives the same logits without materialising a [Q, 256, 256] fp32 map per layer.
__global__ void __launch_bounds__(256)
resize_bilinear_nhwc_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int nb, int H, int W, int C, int h2, int w2) {
  const int vec = C >> 3;
  const long long total = static_cast<long long>(nb) * h2 * w2 * vec;
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int cv = static_cast<int>(idx % vec);
  long long r = idx / vec;
  const int ox = static_cast<int>(r % w2); r /= w2;
  const int oy = static_cast<int>(r % h2);
  const long long n = r / h2;
  const float sh = static_cast<float>(H) / h2, sw = static_cast<float>(W) / w2;
  const float sy = fmaxf((oy + 0.5f) * sh - 0.5f, 0.f), sx = fmaxf((ox + 0.5f) * sw - 0.5f, 0.f);
  const int y0 = min(static_cast<int>(sy), H - 1), x0 = min(static_cast<int>(sx), W - 1);
  const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  const float ly = sy - y0, lx = sx - x0;
  const bf16* base = x + n * H * W * C + cv * 8;
  const uint4 a = *reinterpret_cast<const uint4*>(base + (static_cast<long long>(y0) * W + x0) * C);
  const uint4 b = *reinterpret_cast<const uint4*>(base + (static_cast<long long>(y0) * W + x1) * C);
  const uint4 c = *reinterpret_cast<const uint4*>(base + (static_cast<long long>(y1) * W + x0) * C);
  const uint4 d = *reinterpret_cast<const uint4*>(base + (static_cast<long long>(y1) * W + x1) * C);
  const uint32_t aa[4] = {a.x, a.y, a.z, a.w}, bb[4] = {b.x, b.y, b.z, b.w}, cc[4] = {c.x, c.y, c.z, c.w}, dd[4] = {d.x, d.y, d.z, d.w};
  uint32_t oo[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 fa = unpack_bf16(aa[j]), fb = unpack_bf16(bb[j]), fc = unpack_bf16(cc[j]), fd = unpack_bf16(dd[j]);
    const float v0 = (1 - ly) * ((1 - lx) * fa.x + lx * fb.x) + ly * ((1 - lx) * fc.x + lx * fd.x);
    const float v1 = (1 - ly) * ((1 - lx) * fa.y + lx * fb.y) + ly * ((1 - lx) * fc.y + lx * fd.y);
    oo[j] = pack_bf16(v0, v1);
  }
  *reinterpret_cast<uint4*>(out + ((n * h2 + oy) * w2 + ox) * C + cv * 8) = make_uint4(oo[0], oo[1], oo[2], oo[3]);
}

// direct NHWC conv, one thread per (output pixel, output channel); only for tiny layers
__global__ void conv_direct_kernel(const bf16* __restrict__ x, const bf16* __restrict__ wt, const bf16* __restrict__ bias,
                                   bf16* __restrict__ out, int nb, int h, int w, int cin, int cout, int kh, int kw,
                                   int stride, int ph, int pw, int ho, int wo) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long total = static_cast<long long>(nb) * ho * wo * cout;
  if (idx >= total) return;
  const int co = static_cast<int>(idx % cout);
  long long r = idx / cout;
  const int ox = static_cast<int>(r % wo); r /= wo;
  const int oy = static_cast<int>(r % ho);
  const long long n = r / ho;
  float acc = bias ? __bfloat162float(bias[co]) : 0.f;
  for (int ky = 0; ky < kh; ++ky) {
    const int iy = oy * stride - ph + ky;
    if (iy < 0 || iy >= h) continue;
    for (int kx = 0; kx < kw; ++kx) {
      const int ix = ox * stride - pw + kx;
      if (ix < 0 || ix >= w) continue;
      const bf16* xp = x + ((n * h + iy) * w + ix) * cin;
      const bf16* wp = wt + (static_cast<long long>(co) * kh * kw + ky * kw + kx) * cin;
      for (int ci = 0; ci < cin; ++ci) acc += __bfloat162float(xp[ci]) * __bfloat162float(wp[ci]);
    }
  }
  out[idx] = __float2bfloat16(acc);
}

// ------------------------------------------------------------------ row softmax (VAE AttnBlock)
// out[row, :] = softmax(x[row, :]) ; x fp32 [rows, ldx], out bf16 [rows, ldo]; one CTA per row, online
// max/sum in one read, second read (L1/L2 resident) writes the probabilities.
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ x, long long ldx, bf16* __restrict__ out,
                                                           long long ldo, int n) {
  __shared__ float sm[8], ss[8];
  const float* xr = x + blockIdx.x * ldx;
  bf16* orow = out + blockIdx.x * ldo;
  float m = -INFINITY, s = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) {
    const float v = xr[i];
    // a -inf adds nothing to the sum; taken into the online update while m is still -inf, it would make m - mn NaN
    if (v == -INFINITY) continue;
    const float mn = fmaxf(m, v);
    s = s * __expf(m - mn) + __expf(v - mn);
    m = mn;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float mo = __shfl_xor_sync(0xffffffffu, m, o), so = __shfl_xor_sync(0xffffffffu, s, o);
    const float mn = fmaxf(m, mo);
    s = (m == -INFINITY ? 0.f : s * __expf(m - mn)) + (mo == -INFINITY ? 0.f : so * __expf(mo - mn));
    m = mn;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sm[warp] = m; ss[warp] = s; }
  __syncthreads();
  float gm = -INFINITY;
#pragma unroll
  for (int w = 0; w < 8; ++w) gm = fmaxf(gm, sm[w]);
  float gs = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) gs += sm[w] == -INFINITY ? 0.f : ss[w] * __expf(sm[w] - gm);
  const float inv = 1.0f / gs;
  for (int i = threadIdx.x; i < n; i += 256) orow[i] = __float2bfloat16(__expf(xr[i] - gm) * inv);
}

}  // namespace vb

using namespace vb;

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int vb200_softmax_rows(const float* x, int64_t ldx, void* out, int64_t ldo, int64_t rows, int64_t n,
                                  cudaStream_t stream) {
  VB_CHECK_ARG(x && out && rows >= 0 && n > 0 && ldx >= n && ldo >= n && n < (1ll << 31));
  if (rows == 0) return VB_OK;
  softmax_rows_kernel<<<static_cast<unsigned>(rows), 256, 0, stream>>>(x, ldx, reinterpret_cast<bf16*>(out), ldo,
                                                                       static_cast<int>(n));
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_patchify(const void* pixels, int in_is_fp32, void* out, int64_t nb, int64_t c, int64_t h,
                              int64_t w, int64_t patch, int64_t kpad, cudaStream_t stream) {
  VB_CHECK_ARG(pixels && out && nb > 0 && c > 0 && patch > 0 && h % patch == 0 && w % patch == 0);
  VB_CHECK_ARG(kpad >= c * patch * patch && kpad % 8 == 0);
  const long long total = nb * (h / patch) * (w / patch) * kpad;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  if (in_is_fp32)
    patchify_kernel<float><<<blocks, 256, 0, stream>>>(reinterpret_cast<const float*>(pixels), reinterpret_cast<bf16*>(out), (int)c, (int)h, (int)w, (int)patch, (int)kpad, total);
  else
    patchify_kernel<bf16><<<blocks, 256, 0, stream>>>(reinterpret_cast<const bf16*>(pixels), reinterpret_cast<bf16*>(out), (int)c, (int)h, (int)w, (int)patch, (int)kpad, total);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_vit_embed_ln(const void* patch_out, const void* cls, const void* pos, const void* ln_w,
                                  const void* ln_b, void* out, int64_t nb, int64_t npatch, int64_t d, float eps,
                                  cudaStream_t stream) {
  VB_CHECK_ARG(patch_out && cls && pos && ln_w && ln_b && out && nb > 0 && npatch > 0 && d > 0 && d <= 2048);
  vit_embed_ln_kernel<<<static_cast<unsigned>(nb * (npatch + 1)), 128, 0, stream>>>(
      reinterpret_cast<const bf16*>(patch_out), reinterpret_cast<const bf16*>(cls), reinterpret_cast<const bf16*>(pos),
      reinterpret_cast<const bf16*>(ln_w), reinterpret_cast<const bf16*>(ln_b), reinterpret_cast<bf16*>(out),
      (int)npatch, (int)d, eps);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_upsample2x_nhwc(const void* x, void* out, int64_t nb, int64_t h, int64_t w, int64_t c,
                                     cudaStream_t stream) {
  VB_CHECK_ARG(x && out && nb > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0 && aligned16(x) && aligned16(out));
  const long long total = nb * 2 * h * 2 * w * (c / 8);
  upsample2x_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), (int)h, (int)w, (int)(c / 8), total);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_add_bf16(const void* a, const void* b, void* out, int64_t n, int64_t b_period,
                              cudaStream_t stream) {
  VB_CHECK_ARG(a && b && out && n >= 0 && n % 8 == 0 && b_period % 8 == 0);
  VB_CHECK_ARG(aligned16(a) && aligned16(b) && aligned16(out));
  if (n == 0) return VB_OK;
  add_kernel<<<static_cast<unsigned>((n / 8 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const uint4*>(a), reinterpret_cast<const uint4*>(b), reinterpret_cast<uint4*>(out), n / 8,
      b_period / 8);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_add_rowgroup(const void* x, const void* table, void* out, int64_t rows, int64_t d,
                                  int64_t group_rows, int64_t period, cudaStream_t stream) {
  VB_CHECK_ARG(x && table && out && rows >= 0 && d > 0 && d % 8 == 0 && group_rows > 0 && period > 0);
  VB_CHECK_ARG(aligned16(x) && aligned16(table) && aligned16(out));
  if (rows == 0) return VB_OK;
  const long long nvec = rows * (d / 8);
  add_rowgroup_kernel<<<static_cast<unsigned>((nvec + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const uint4*>(x), reinterpret_cast<const uint4*>(table), reinterpret_cast<uint4*>(out), nvec,
      static_cast<int>(d / 8), group_rows, period);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_cfg_combine(const void* y, const void* u, void* out, float scale, int64_t n,
                                 cudaStream_t stream) {
  VB_CHECK_ARG(y && u && out && n >= 0);
  if (n == 0) return VB_OK;
  cfg_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const float*>(y), reinterpret_cast<const float*>(u), reinterpret_cast<float*>(out), scale, n);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_region_mask_pool(const void* feats, const float* boxes, void* out, int64_t B, int64_t grid,
                                      int64_t c, int64_t image_size, cudaStream_t stream) {
  VB_CHECK_ARG(feats && boxes && out && B > 0 && grid > 0 && c > 0 && image_size > 0);
  VB_CHECK_ARG(grid * grid * sizeof(float) <= 40 * 1024);   // cell weights live in (default-limit) dynamic shared memory
  dim3 g(static_cast<unsigned>((c + 255) / 256), static_cast<unsigned>(B));
  region_pool_kernel<<<g, 256, grid * grid * sizeof(float), stream>>>(
      reinterpret_cast<const bf16*>(feats), boxes, reinterpret_cast<bf16*>(out), (int)grid, (int)c, (int)image_size);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_seem_attn_mask(const float* mask_logits, uint8_t* out_mask, int64_t Q, int64_t H, int64_t W,
                                    int64_t h2, int64_t w2, cudaStream_t stream) {
  VB_CHECK_ARG(mask_logits && out_mask && Q > 0 && H > 0 && W > 0 && h2 > 0 && w2 > 0);
  seem_mask_kernel<<<static_cast<unsigned>(Q), 256, 0, stream>>>(mask_logits, out_mask, (int)H, (int)W, (int)h2, (int)w2);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_resize_bilinear_nhwc(const void* x, void* out, int64_t nb, int64_t H, int64_t W, int64_t C, int64_t h2,
                                          int64_t w2, cudaStream_t stream) {
  VB_CHECK_ARG(x && out && nb > 0 && H > 0 && W > 0 && C > 0 && (C % 8) == 0 && h2 > 0 && w2 > 0);
  VB_CHECK_ARG(aligned16(x) && aligned16(out));
  const long long total = nb * h2 * w2 * (C / 8);
  resize_bilinear_nhwc_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(out), (int)nb, (int)H, (int)W, (int)C, (int)h2, (int)w2);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

extern "C" int vb200_conv_nhwc_direct(const void* X, const void* Wt, const void* bias, void* out, int64_t nb,
                                      int64_t h, int64_t w, int64_t cin, int64_t cout, int kh, int kw, int stride,
                                      int pad_h, int pad_w, cudaStream_t stream) {
  VB_CHECK_ARG(X && Wt && out && nb > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && stride > 0);
  const int ho = static_cast<int>((h + 2 * pad_h - kh) / stride + 1), wo = static_cast<int>((w + 2 * pad_w - kw) / stride + 1);
  const long long total = nb * ho * wo * cout;
  conv_direct_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const bf16*>(X), reinterpret_cast<const bf16*>(Wt), reinterpret_cast<const bf16*>(bias),
      reinterpret_cast<bf16*>(out), (int)nb, (int)h, (int)w, (int)cin, (int)cout, kh, kw, stride, pad_h, pad_w, ho, wo);
  VB_LAUNCH_CHECK();
  return VB_OK;
}
