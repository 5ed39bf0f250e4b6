// vitron_b200 — NF4 weight-streaming GEMM for M <= 32 tokens, and the NF4 -> bf16 dequantiser.
//
//   out[M, N'] = epilogue( rowscale ⊙ (X~[M, K] · W_tab[N, K]^T) ),  M <= 32
//   X~[m, k] = bf16_rn(float(X[m, k]) * kscale[k])   (X itself without kscale)
//   W_tab[n, k] = bf16_rn(nf4[code(n, k)]) * float(scale(n, k / 64)), the scale applied in fp32 to each 64-block's sum
//
// W_tab is not the format's W_eff = nf4[code] * scale (vitron_b200/nf4.py): the table holds the NF4 values rounded to
// bf16, which moves 13 of the 16 by up to 3.1e-3 relative (code 2), far below NF4's own quantisation error. Keeping the
// fp32 values would cost the bf16x2 table lookup that feeds the mma directly. The dequantiser below rounds the other
// product, bf16_rn(nf4[code] * scale * kscale[k]). tests/test_nf4_kernels_gpu.py pins the kernel against W_tab and bounds
// its distance to W_eff.
//
// Decode is bound by weight bytes; 4-bit codes + one fp16 scale per (row, 64-block) stream 0.53 bytes per weight
// instead of 2. The kernel follows gemv_bf16_kernel (gemv.cu): persistent, 2 CTAs per SM, each CTA owns 16 (32 for the
// packed-GLU layout) output features, its 8 warps split K, weights stream with 16-byte loads on the non-allocating path
// and are requested before the PDL dependency wait, the pipeline runs across tiles, and the products run on mma.sync
// m16n8k16 with the weights as A. Per 64-block a thread owns the same k positions as in gemv.cu ([8t, 8t+8) and
// [32+8t, 32+8t+8)); the codes are stored so that those 16 codes of two consecutive blocks are one 16-byte load, each
// byte holding a k pair (low nibble = lower k). A byte maps to its bf16x2 A-fragment register through a 256-entry
// table in shared memory with one copy per lane (word [byte][lane]: every lookup hits the lane's own bank). The partial
// products of a 64-block are accumulated unscaled and multiplied by the block's scale once per row and block.
#include "common.cuh"
#include "vitron_b200.h"
#include <cuda_fp16.h>

namespace vb {

// bitsandbytes' NF4 code (vitron_b200/nf4.py NF4)
__constant__ float kNF4[16] = {-1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f,
                               -0.28444138169288635f, -0.18477343022823334f, -0.09105003625154495f, 0.0f,
                               0.07958029955625534f, 0.16093020141124725f, 0.24611230194568634f, 0.33791524171829224f,
                               0.44070982933044434f, 0.5626170039176941f, 0.7229568362236023f, 1.0f};

struct Nf4Params {
  const uint8_t* codes; long long ldc;   // bytes per row: 64 per 128 k (K rounded up to 128)
  const __half* scales; long long lds;   // K / 64 per row
  const float* kscale;
  const bf16* X; long long ldx;
  void* out; long long ldo;
  int M, N, K;
  const bf16* bias; const bf16* rowbias; int rowbias_rows;
  const bf16* residual; long long ldr;
  float alpha; int act, glu, out_fp32;
  const float* rowscale; float rms_eps;
};

__device__ __forceinline__ float nf4_act(float x, int act) {
  switch (act) {
    case VB_ACT_GELU: return gelu_erf(x);
    case VB_ACT_QUICK_GELU: return quick_gelu(x);
    case VB_ACT_RELU: return fmaxf(x, 0.f);
    case VB_ACT_SILU: return silu(x);
    default: return x;
  }
}

__device__ __forceinline__ void nf4_mma(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                        uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint4 nf4_ldg_stream(const uint8_t* p, bool ok) {
  uint4 v = make_uint4(0, 0, 0, 0);
  if (ok) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

__device__ __forceinline__ uint4 nf4_ldg_x(const void* p, bool ok) {
  uint4 v = make_uint4(0, 0, 0, 0);
  if (ok) v = __ldg(reinterpret_cast<const uint4*>(p));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  const bf162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}

template <int NT>
constexpr int nf4_smem_bytes() { return (256 * 32 + 2 * 8 * 16 * (NT * 8 + 1)) * 4; }

// ROWS = 16 or 32 output features per tile; NT = 1, 2 or 4 token tiles of 8 (M <= 8, 16, 32).
template <int ROWS, int NT>
__global__ void __launch_bounds__(256, 2) gemv_nf4_kernel(const Nf4Params p) {
  constexpr int WARPS = 8;
  constexpr int RG = ROWS / 16;        // row groups per tile
  constexpr int KS = WARPS / RG;       // k-slices per row group
  constexpr int G = NT == 4 ? 1 : 2;   // 128-wide superchunks (16-byte loads per row) per load group (fewer registers at NT = 4)
  constexpr int TOK = NT * 8;
  constexpr int RS = TOK + 1;          // padded row of the reduction buffer
  extern __shared__ __align__(16) uint32_t nf4_smem[];
  uint32_t* lut = nf4_smem;                                         // [256 byte values][32 lanes] bf16x2
  float* red = reinterpret_cast<float*>(nf4_smem + 256 * 32);       // [2 parity][WARPS][16][RS]
  __shared__ float red_sq[WARPS][TOK];
  __shared__ float rstd_s[TOK];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int rg = warp % RG, ks = warp / RG;
  const int ntiles = (p.N + ROWS - 1) / ROWS;

  const int chunks = p.K / 64;                     // scale blocks per row
  const int nsc = (chunks + 1) / 2;                // superchunks per row
  const int base = nsc / KS, rem = nsc % KS;
  const int s0 = ks * base + min(ks, rem);
  const int s1 = s0 + base + (ks < rem ? 1 : 0);
  const int ngroups = (s1 - s0 + G - 1) / G;
  const int npairs = (ngroups + 1) / 2;

  const bool do_rms = p.rms_eps > 0.f && p.rowscale == nullptr;
  float sq[NT];
#pragma unroll
  for (int j = 0; j < NT; ++j) sq[j] = 0.f;

  struct Buf { uint4 w[G][2]; unsigned short sc[2]; };  // codes of rows g, g + 8; lane t's scale of block 2 * G * grp + t
  auto load_group = [&](Buf& bf, int tile, int grp) {
    const int row0 = tile * ROWS + rg * 16;
    const int ra = min(row0 + g, p.N - 1), rb = min(row0 + g + 8, p.N - 1);  // clamped rows are masked in the epilogue
    const uint8_t* wa = p.codes + static_cast<long long>(ra) * p.ldc + 16 * t;
    const uint8_t* wb = p.codes + static_cast<long long>(rb) * p.ldc + 16 * t;
    const bool live = tile < ntiles;
#pragma unroll
    for (int v = 0; v < G; ++v) {
      const int s = s0 + grp * G + v;
      const bool in = live && s < s1;
      bf.w[v][0] = nf4_ldg_stream(wa + s * 64, in);
      bf.w[v][1] = nf4_ldg_stream(wb + s * 64, in);
    }
    const int c = 2 * (s0 + grp * G) + t;
    const bool okc = live && t < 2 * G && c < 2 * s1 && c < chunks;
    const unsigned short* sp = reinterpret_cast<const unsigned short*>(p.scales);
    bf.sc[0] = okc ? __ldg(sp + static_cast<long long>(ra) * p.lds + c) : 0;
    bf.sc[1] = okc ? __ldg(sp + static_cast<long long>(rb) * p.lds + c) : 0;
  };

  float acc[NT][4];
  auto compute_group = [&](const Buf& bf, int grp, bool first_tile) {
#pragma unroll
    for (int v = 0; v < G; ++v) {
      const int s = s0 + grp * G + v;
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int c = 2 * s + u;
        const bool ok = s < s1 && c < chunks;
        const int k0 = c * 64 + 8 * t, k1 = k0 + 32;
        const int src = (lane & ~3) | (2 * v + u);
        const float sa = __half2float(__ushort_as_half(__shfl_sync(0xffffffffu, bf.sc[0], src)));
        const float sb = __half2float(__ushort_as_half(__shfl_sync(0xffffffffu, bf.sc[1], src)));
        const uint32_t la[2] = {u ? bf.w[v][0].z : bf.w[v][0].x, u ? bf.w[v][0].w : bf.w[v][0].y};
        const uint32_t lb[2] = {u ? bf.w[v][1].z : bf.w[v][1].x, u ? bf.w[v][1].w : bf.w[v][1].y};
        uint32_t al[8], ah[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          al[i] = lut[(((la[i >> 2] >> (8 * (i & 3))) & 0xffu) << 5) | lane];
          ah[i] = lut[(((lb[i >> 2] >> (8 * (i & 3))) & 0xffu) << 5) | lane];
        }
        float kv[16];
        if (p.kscale) {
          const float4 q0 = ok ? __ldg(reinterpret_cast<const float4*>(p.kscale + k0)) : make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 q1 = ok ? __ldg(reinterpret_cast<const float4*>(p.kscale + k0 + 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 q2 = ok ? __ldg(reinterpret_cast<const float4*>(p.kscale + k1)) : make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 q3 = ok ? __ldg(reinterpret_cast<const float4*>(p.kscale + k1 + 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
          kv[0] = q0.x; kv[1] = q0.y; kv[2] = q0.z; kv[3] = q0.w; kv[4] = q1.x; kv[5] = q1.y; kv[6] = q1.z; kv[7] = q1.w;
          kv[8] = q2.x; kv[9] = q2.y; kv[10] = q2.z; kv[11] = q2.w; kv[12] = q3.x; kv[13] = q3.y; kv[14] = q3.z; kv[15] = q3.w;
        }
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const int tok = g + 8 * j;
          const bf16* xr = p.X + static_cast<long long>(min(tok, p.M - 1)) * p.ldx;
          const bool xok = ok && tok < p.M;
          const uint4 xa = nf4_ldg_x(xr + k0, xok), xb = nf4_ldg_x(xr + k1, xok);
          uint32_t b[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
          if (do_rms && first_tile && rg == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { const float2 f = unpack_bf16(b[i]); sq[j] += f.x * f.x + f.y * f.y; }
          }
          if (p.kscale) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float2 f = unpack_bf16(b[i]);
              b[i] = pack_bf16x2(f.x * kv[2 * i], f.y * kv[2 * i + 1]);
            }
          }
          float tmp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int i = 0; i < 4; ++i) nf4_mma(tmp, al[2 * i], ah[2 * i], al[2 * i + 1], ah[2 * i + 1], b[2 * i], b[2 * i + 1]);
          acc[j][0] = fmaf(tmp[0], sa, acc[j][0]);
          acc[j][1] = fmaf(tmp[1], sa, acc[j][1]);
          acc[j][2] = fmaf(tmp[2], sb, acc[j][2]);
          acc[j][3] = fmaf(tmp[3], sb, acc[j][3]);
        }
      }
    }
  };

  Buf buf0, buf1;
  pdl_trigger();
  // codes and scales never depend on the previous kernel: two groups are requested before the dependency wait
  load_group(buf0, blockIdx.x, 0);
  load_group(buf1, blockIdx.x, 1);
  for (int i = threadIdx.x; i < 256 * 32; i += 256) {
    const int byte = i >> 5;
    lut[i] = pack_bf16x2(kNF4[byte & 15], kNF4[byte >> 4]);
  }
  __syncthreads();
  pdl_wait();

  const bool glu = p.glu != VB_GLU_NONE;
  const int out_cols = glu ? ROWS / 2 : ROWS;            // ROWS == 32 when glu
  const int n_out_total = glu ? p.N / 2 : p.N;
  int par = 0;
  bool first = true;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
#pragma unroll
    for (int i = 0; i < NT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    for (int pr = 0; pr < npairs; ++pr) {
      const bool last = pr + 1 == npairs;                 // then prefetch the first two groups of the NEXT tile
      compute_group(buf0, 2 * pr, first);
      if (!last) load_group(buf0, tile, 2 * pr + 2); else load_group(buf0, tile + gridDim.x, 0);
      compute_group(buf1, 2 * pr + 1, first);             // groups past the slice carry zero operands
      if (!last) load_group(buf1, tile, 2 * pr + 3); else load_group(buf1, tile + gridDim.x, 1);
    }
    // ---- cross-warp (k-slice) reduction: red[par][warp][feature 0..15][token]
    float* rw = red + ((par * WARPS + warp) * 16) * RS;
#pragma unroll
    for (int i = 0; i < NT; ++i) {
      rw[g * RS + i * 8 + 2 * t] = acc[i][0];
      rw[g * RS + i * 8 + 2 * t + 1] = acc[i][1];
      rw[(g + 8) * RS + i * 8 + 2 * t] = acc[i][2];
      rw[(g + 8) * RS + i * 8 + 2 * t + 1] = acc[i][3];
    }
    if (do_rms && first) {
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        sq[j] += __shfl_xor_sync(0xffffffffu, sq[j], 1);
        sq[j] += __shfl_xor_sync(0xffffffffu, sq[j], 2);
        if (t == 0) red_sq[warp][8 * j + g] = sq[j];
      }
    }
    __syncthreads();
    if (do_rms && first) {
      if (threadIdx.x < TOK) {
        float ss = 0.f;
#pragma unroll
        for (int s2 = 0; s2 < KS; ++s2) ss += red_sq[s2 * RG][threadIdx.x];  // row-group-0 warps cover every k once
        rstd_s[threadIdx.x] = rsqrtf(ss / p.K + p.rms_eps);
      }
      __syncthreads();
    }
    // ---- epilogue: one thread per (token, output column of this tile)
    const float* rp = red + par * WARPS * 16 * RS;
    for (int item = threadIdx.x; item < p.M * out_cols; item += 256) {
      const int tok = item / out_cols, j = item % out_cols;
      const int fa = j, fb = j + 16;                       // packed GLU layout: [16 x a | 16 x b]
      const int na = tile * ROWS + fa;                      // accumulator column (weight row)
      const int oc = glu ? tile * (ROWS / 2) + j : na;
      if (oc >= n_out_total) continue;
      float va = 0.f, vb_ = 0.f;
#pragma unroll
      for (int s2 = 0; s2 < KS; ++s2) {
        va += rp[((s2 * RG + fa / 16) * 16 + fa % 16) * RS + tok];
        if (glu) vb_ += rp[((s2 * RG + (fb / 16) % RG) * 16 + fb % 16) * RS + tok];
      }
      if (do_rms) { const float rs = rstd_s[tok]; va *= rs; vb_ *= rs; }
      else if (p.rowscale) { const float rs = p.rowscale[tok]; va *= rs; vb_ *= rs; }
      if (p.bias) {
        va += __bfloat162float(p.bias[na]);
        if (glu) vb_ += __bfloat162float(p.bias[na + 16]);
      }
      if (p.rowbias) {
        const bf16* rbp = p.rowbias + (tok / p.rowbias_rows) * static_cast<long long>(p.N);
        va += __bfloat162float(rbp[na]);
        if (glu) vb_ += __bfloat162float(rbp[na + 16]);
      }
      float r;
      if (p.glu == VB_GLU_SWIGLU) r = silu(va) * vb_;
      else if (p.glu == VB_GLU_GEGLU) r = va * gelu_erf(vb_);
      else r = nf4_act(va, p.act);
      if (p.residual) r = __bfloat162float(p.residual[tok * p.ldr + oc]) + p.alpha * r;
      else r *= p.alpha;
      if (p.out_fp32) reinterpret_cast<float*>(p.out)[tok * p.ldo + oc] = r;
      else reinterpret_cast<bf16*>(p.out)[tok * p.ldo + oc] = __float2bfloat16(r);
    }
    par ^= 1;
    first = false;
  }
}

// One thread per 16-byte code unit (32 weights of one row): out[n, k] = bf16_rn((nf4[code] * scale) * kscale[k]),
// each product rounded to fp32 in that order (the statement of vitron_b200/nf4.py, bit for bit).
__global__ void __launch_bounds__(256) nf4_dequant_kernel(const uint8_t* __restrict__ codes, long long ldc,
                                                           const __half* __restrict__ scales, long long lds,
                                                           const float* __restrict__ kscale, bf16* __restrict__ out,
                                                           int N, int K) {
  __shared__ float tab[16];
  if (threadIdx.x < 16) tab[threadIdx.x] = kNF4[threadIdx.x];
  __syncthreads();
  pdl_trigger();
  const int chunks = K / 64, nsc = (chunks + 1) / 2;
  const long long unit = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool live = unit < static_cast<long long>(N) * nsc * 4;
  const int n = live ? static_cast<int>(unit / (nsc * 4)) : 0;
  const int s = live ? static_cast<int>((unit / 4) % nsc) : 0, t = static_cast<int>(unit % 4);
  const uint4 w = live ? __ldg(reinterpret_cast<const uint4*>(codes + n * ldc + s * 64 + 16 * t)) : make_uint4(0, 0, 0, 0);
  pdl_wait();   // out may be a workspace that the previous kernel still reads
  if (!live) return;
  const uint32_t words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int c = 2 * s + u;
    if (c >= chunks) break;
    const float sc = __half2float(scales[static_cast<long long>(n) * lds + c]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k = c * 64 + 32 * h + 8 * t;
      const uint32_t word = words[2 * u + h];
      uint32_t o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t byte = (word >> (8 * i)) & 0xffu;
        float lo = __fmul_rn(tab[byte & 15], sc), hi = __fmul_rn(tab[byte >> 4], sc);
        if (kscale) { lo = __fmul_rn(lo, kscale[k + 2 * i]); hi = __fmul_rn(hi, kscale[k + 2 * i + 1]); }
        o[i] = pack_bf16x2(lo, hi);
      }
      *reinterpret_cast<uint4*>(out + static_cast<long long>(n) * K + k) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

template <int ROWS, int NT>
static cudaError_t launch_nf4(const Nf4Params& p, unsigned grid, cudaStream_t stream) {
  static bool attr_set = false;   // > 48 KB of dynamic shared memory needs the opt-in once per kernel
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemv_nf4_kernel<ROWS, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         nf4_smem_bytes<NT>());
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  return vb_launch(gemv_nf4_kernel<ROWS, NT>, dim3(grid), dim3(256), nf4_smem_bytes<NT>(), stream, p);
}

}  // namespace vb

using namespace vb;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int vb200_gemm_nf4(const void* A, int64_t lda, const void* codes, const void* scales, const float* kscale,
                              void* out, int64_t ldo, int64_t M, int64_t N, int64_t K, const vb_epilogue* epi,
                              cudaStream_t stream) {
  VB_CHECK_ARG(A && codes && scales && out && epi);
  VB_CHECK_ARG(M > 0 && N > 0 && K > 0 && (K % 64) == 0);
  VB_CHECK_ARG((lda % 8) == 0 && lda >= K && aligned16(A) && aligned16(codes) && (kscale == nullptr || aligned16(kscale)));
  VB_CHECK_ARG(ldo >= (epi->glu != VB_GLU_NONE ? N / 2 : N));
  if (epi->glu != VB_GLU_NONE && (N % 32) != 0) return VB_ERR_ARG;
  if (epi->act < VB_ACT_NONE || epi->act > VB_ACT_SILU || epi->glu < VB_GLU_NONE || epi->glu > VB_GLU_GEGLU) return VB_ERR_ARG;
  if (M > 32) return VB_ERR_UNSUPPORTED;
  Nf4Params p;
  p.codes = reinterpret_cast<const uint8_t*>(codes); p.ldc = (K + 127) / 128 * 64;
  p.scales = reinterpret_cast<const __half*>(scales); p.lds = K / 64;
  p.kscale = kscale;
  p.X = reinterpret_cast<const bf16*>(A); p.ldx = lda;
  p.out = out; p.ldo = ldo;
  p.M = static_cast<int>(M); p.N = static_cast<int>(N); p.K = static_cast<int>(K);
  p.bias = reinterpret_cast<const bf16*>(epi->bias);
  p.rowbias = reinterpret_cast<const bf16*>(epi->rowbias);
  p.rowbias_rows = epi->rowbias_rows > 0 ? static_cast<int>(epi->rowbias_rows) : 1;
  p.residual = reinterpret_cast<const bf16*>(epi->residual); p.ldr = epi->ldr;
  p.alpha = epi->alpha; p.act = epi->act; p.glu = epi->glu; p.out_fp32 = epi->out_fp32;
  p.rowscale = epi->rowscale; p.rms_eps = epi->rms_eps;
  // tile choice as in gemv.cu: 32-row CTAs for the packed GLU layout or when 16-row CTAs would exceed ~4 per SM
  const bool rows32 = epi->glu != VB_GLU_NONE || (N / 16 > 6LL * vb_num_sms());
  const unsigned tiles = static_cast<unsigned>((N + (rows32 ? 31 : 15)) / (rows32 ? 32 : 16));
  const unsigned cap = 2u * static_cast<unsigned>(vb_num_sms());
  const unsigned grid = tiles < cap ? tiles : cap;
  cudaError_t err;
  if (M <= 8) err = rows32 ? launch_nf4<32, 1>(p, grid, stream) : launch_nf4<16, 1>(p, grid, stream);
  else if (M <= 16) err = rows32 ? launch_nf4<32, 2>(p, grid, stream) : launch_nf4<16, 2>(p, grid, stream);
  else err = rows32 ? launch_nf4<32, 4>(p, grid, stream) : launch_nf4<16, 4>(p, grid, stream);
  if (err != cudaSuccess) { vb_set_last_error(err); return VB_ERR_CUDA; }
  return VB_OK;
}

extern "C" int vb200_nf4_dequant(const void* codes, const void* scales, const float* kscale, void* out, int64_t N,
                                 int64_t K, cudaStream_t stream) {
  VB_CHECK_ARG(codes && scales && out);
  VB_CHECK_ARG(N > 0 && K > 0 && (K % 64) == 0);
  VB_CHECK_ARG(aligned16(codes) && aligned16(out));
  const long long units = N * ((K / 64 + 1) / 2) * 4;
  const unsigned grid = static_cast<unsigned>((units + 255) / 256);
  cudaError_t err = vb_launch(nf4_dequant_kernel, dim3(grid), dim3(256), 0, stream,
                              reinterpret_cast<const uint8_t*>(codes), (K + 127) / 128 * 64,
                              reinterpret_cast<const __half*>(scales), K / 64, kscale, reinterpret_cast<bf16*>(out),
                              static_cast<int>(N), static_cast<int>(K));
  if (err != cudaSuccess) { vb_set_last_error(err); return VB_ERR_CUDA; }
  return VB_OK;
}
