// vitron_b200 — pieces shared by the wgmma GEMM / implicit-GEMM convolution kernel (gemm_v2.cuh) and its host side
// (gemm.cu: planning, split-K reduce). See gemm_v2.cuh for the design notes.
#pragma once
#include "common.cuh"
#include "vitron_b200.h"

namespace vb {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int GEMM_THREADS = 3 * 128;  // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + epilogue, 64 tile rows each
constexpr int SMEM_LIMIT = 227 * 1024;

struct GemmParams {
  int M, N;           // logical output extent (rows of A-space, rows of B)
  int num_k_blocks;   // k-steps of BLOCK_K (conv: taps * cin_chunks)
  int splits;         // split-K factor (>=1)
  int m_blocks, n_blocks;
  // ---- A addressing
  int a_mode;         // 0: 2-D matrix, 1: NHWC conv
  int cin_chunks;     // conv: BLOCK_K chunks per tap
  int kw;             // conv: kernel width (tap -> dy = tap / kw, dx = tap % kw)
  int stride, pad_h, pad_w;
  int tw, th, tn;     // conv: output-pixel tile (tw*th*tn <= 128)
  int wo, ho, nb;     // conv: output width / height / images
  int tiles_w, tiles_h;
  uint32_t a_box_bytes;
  // ---- epilogue
  void* out;          // bf16 or fp32 [rows, ldo]
  long long ldo;
  const bf16* bias;      // [N] or null
  const bf16* rowbias;   // [groups, N] or null; group = out_row / rowbias_rows
  int rowbias_rows;
  const bf16* residual;  // [rows, ldr] or null; out = residual + alpha * v
  long long ldr;
  float alpha;
  const float* rowscale;  // fp32 per output row (C orientation) or null
  int act;            // VB_ACT_*
  int glu;            // VB_GLU_*
  int out_fp32;
  int swap;           // accumulator rows are output columns (decode / tiny-M path) -> workspace
  float* ws;          // split-K / swap workspace [splits, rows_c, cols_c] fp32
  long long ws_split_stride;
  long long ws_ld;
  int dbg;            // measurement aid (vb200_set_gemm_debug): bit 0 = the epilogue stores nothing
};

__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case VB_ACT_GELU: return gelu_erf_fast(x);  // exact-erf GELU, |erf error| <= 1.5e-7, straight-line (erff's branches
                                                // made an M = 65536, N = 768 GELU epilogue ALU-bound: 274 us vs ~40)
    case VB_ACT_QUICK_GELU: return quick_gelu(x);
    case VB_ACT_RELU: return fmaxf(x, 0.f);
    case VB_ACT_SILU: return silu(x);
    default: return x;
  }
}

// One 8-wide output item of the split-K finalisation: out[row, oc..oc+8) = epi(sum_s ws[s, row, cols]).
// Partials are read with ld.global.cg (L2) because they were written by other CTAs.
__device__ __forceinline__ void reduce_item(const float* __restrict__ ws, int splits, long long split_stride,
                                            long long ws_ld, int row, int oc, int ncols, void* out, long long ldo,
                                            const bf16* __restrict__ bias, const bf16* __restrict__ rowbias,
                                            int rowbias_rows, const bf16* __restrict__ residual, long long ldr,
                                            float alpha, int act, int glu, int out_fp32,
                                            const float* __restrict__ rowscale = nullptr) {
  const int n_out_total = glu != VB_GLU_NONE ? ncols / 2 : ncols;
  int ca = oc, cb = -1;
  if (glu != VB_GLU_NONE) {
    ca = (oc / 16) * 32 + (oc % 16);
    cb = ca + 16;
  }
  float a[8], b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = b[j] = 0.f;
  const bool vec = (oc + 8 <= n_out_total) && ((ws_ld & 3) == 0);
  for (int s = 0; s < splits; ++s) {
    const float* src = ws + s * split_stride + row * ws_ld;
    if (vec) {
      const float4 x0 = __ldcg(reinterpret_cast<const float4*>(src + ca));
      const float4 x1 = __ldcg(reinterpret_cast<const float4*>(src + ca + 4));
      a[0] += x0.x; a[1] += x0.y; a[2] += x0.z; a[3] += x0.w;
      a[4] += x1.x; a[5] += x1.y; a[6] += x1.z; a[7] += x1.w;
      if (cb >= 0) {
        const float4 y0 = __ldcg(reinterpret_cast<const float4*>(src + cb));
        const float4 y1 = __ldcg(reinterpret_cast<const float4*>(src + cb + 4));
        b[0] += y0.x; b[1] += y0.y; b[2] += y0.z; b[3] += y0.w;
        b[4] += y1.x; b[5] += y1.y; b[6] += y1.z; b[7] += y1.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (oc + j < n_out_total) {
          a[j] += __ldcg(src + ca + j);
          if (cb >= 0) b[j] += __ldcg(src + cb + j);
        }
      }
    }
  }
  const bf16* rb = rowbias ? rowbias + (row / rowbias_rows) * static_cast<long long>(ncols) : nullptr;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    v[j] = 0.f;
    if (oc + j >= n_out_total) continue;
    float va = a[j], vb_ = b[j];
    if (rowscale) { const float rs = rowscale[row]; va *= rs; vb_ *= rs; }
    if (bias) {
      va += __bfloat162float(bias[ca + j]);
      if (cb >= 0) vb_ += __bfloat162float(bias[cb + j]);
    }
    if (rb) {
      va += __bfloat162float(rb[ca + j]);
      if (cb >= 0) vb_ += __bfloat162float(rb[cb + j]);
    }
    float r;
    if (glu == VB_GLU_SWIGLU) r = silu(va) * vb_;
    else if (glu == VB_GLU_GEGLU) r = va * gelu_erf(vb_);
    else r = apply_act(va, act);
    if (residual) r = __bfloat162float(residual[row * ldr + oc + j]) + alpha * r;
    else r *= alpha;
    v[j] = r;
  }
  if (out_fp32) {
    float* dst = reinterpret_cast<float*>(out) + row * ldo + oc;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (oc + j < n_out_total) dst[j] = v[j];
  } else {
    bf16* dst = reinterpret_cast<bf16*>(out) + row * ldo + oc;
    if (oc + 8 <= n_out_total && (ldo & 7) == 0) {
      *reinterpret_cast<uint4*>(dst) = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]),
                                                  pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (oc + j < n_out_total) dst[j] = __float2bfloat16(v[j]);
    }
  }
}

struct TileCoord {
  int m_blk, n_blk, split;
};

__device__ __forceinline__ TileCoord decode_work(const GemmParams& p, int unit) {
  TileCoord t;
  int tile = unit / p.splits;
  t.split = unit - tile * p.splits;
  // grouped rasterisation: 16 m-blocks wide so a wave of CTAs re-uses A and B tiles through L2
  const int GROUP_M = 16;
  int per_group = GROUP_M * p.n_blocks;
  int group = tile / per_group;
  int first_m = group * GROUP_M;
  int gsize = min(p.m_blocks - first_m, GROUP_M);
  int in_group = tile - group * per_group;
  t.m_blk = first_m + in_group % gsize;
  t.n_blk = in_group / gsize;
  return t;
}

__device__ __forceinline__ void split_range(const GemmParams& p, int split, int& k0, int& k1) {
  int base = p.num_k_blocks / p.splits, rem = p.num_k_blocks % p.splits;
  k0 = split * base + min(split, rem);
  k1 = k0 + base + (split < rem ? 1 : 0);
}

}  // namespace vb
