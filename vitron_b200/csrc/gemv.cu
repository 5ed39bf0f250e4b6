// vitron_b200 — weight-streaming GEMM for M <= 16 tokens (the decode step, region MLP, time embeds).
//
//   out[M, N'] = epilogue( X[M, K] · W[N, K]^T ),  M <= 16
//
// At M = 8 every weight byte is used for 8 FMAs: the op is HBM-bound (13 GB of Vicuna-7B weights per
// decoded token), so the design goal is bytes in flight, not tensor throughput: no TMA
// prologue, no split-K workspace, one launch with the epilogue fused. Each CTA owns 16 (or 32, for
// the packed-GLU layout) consecutive output features and the whole K range; its 8 warps split K,
// stream their weight rows straight from global memory with 16-byte loads (2 x 64-byte segments
// per row per step, 8 loads in flight per thread), multiply on the legacy m16n8k16 tensor path
// (weights = A, tokens = B; the k order inside a 64-chunk is permuted identically on both
// operands so that each thread's fragment is contiguous in memory), and reduce across warps in smem.
// Replaces the same nn.Linear call sites as gemm.cu for tiny M.
#include "common.cuh"
#include "vitron_b200.h"
#include <type_traits>

namespace vb {

struct GemvParams {
  const bf16* W; long long ldw;
  const bf16* X; long long ldx;
  void* out; long long ldo;
  int M, N, K;
  const bf16* bias; const bf16* rowbias; int rowbias_rows;
  const bf16* residual; long long ldr;
  float alpha; int act, glu, out_fp32;
  const float* rowscale; float rms_eps;
};

__device__ __forceinline__ float gemv_act(float x, int act) {
  switch (act) {
    case VB_ACT_GELU: return gelu_erf(x);
    case VB_ACT_QUICK_GELU: return quick_gelu(x);
    case VB_ACT_RELU: return fmaxf(x, 0.f);
    case VB_ACT_SILU: return silu(x);
    default: return x;
  }
}

__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                         uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint4 ldg_stream(const bf16* p, bool ok) {
  uint4 v = make_uint4(0, 0, 0, 0);
  if (ok) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ uint4 ldg_cached(const bf16* p, bool ok) {
  uint4 v = make_uint4(0, 0, 0, 0);
  if (ok) v = __ldg(reinterpret_cast<const uint4*>(p));
  return v;
}

// ROWS = 16 or 32 output features per tile; NT = 1 (M <= 8) or 2 (M <= 16) token tiles of 8.
// Persistent: grid = 2 CTAs per SM, each CTA walks tiles blockIdx.x, +gridDim.x, ... and keeps its weight
// load pipeline running ACROSS tiles (the first group of the next tile is requested before the cross-warp
// reduction / epilogue of the current one), so there is no per-tile ramp-up or drain.
template <int ROWS, int NT>
__global__ void __launch_bounds__(256, 2) gemv_bf16_kernel(const GemvParams p) {
  constexpr int WARPS = 8;
  constexpr int RG = ROWS / 16;        // row groups per tile
  constexpr int KS = WARPS / RG;       // k-slices per row group
  constexpr int G = 2;                 // 64-wide k-chunks per load group
  __shared__ float red[2][WARPS][16][NT * 8 + 1];  // double-buffered by tile parity
  __shared__ float red_sq[WARPS][NT * 8];
  __shared__ float rstd_s[NT * 8];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int rg = warp % RG, ks = warp / RG;
  const int ntiles = (p.N + ROWS - 1) / ROWS;
  const bf16* x0 = p.X + static_cast<long long>(min(g, p.M - 1)) * p.ldx;
  const bf16* x1 = p.X + static_cast<long long>(min(g + 8, p.M - 1)) * p.ldx;
  const bool x0ok = g < p.M, x1ok = (NT == 2) && (g + 8 < p.M);

  const int chunks = (p.K + 63) / 64;
  const int base = chunks / KS, rem = chunks % KS;
  const int c0 = ks * base + min(ks, rem);
  const int c1 = c0 + base + (ks < rem ? 1 : 0);
  const int ngroups = (c1 - c0 + G - 1) / G;
  const int npairs = (ngroups + 1) / 2;

  const bool do_rms = p.rms_eps > 0.f && p.rowscale == nullptr;
  float sq0 = 0.f, sq1 = 0.f;

  struct Buf { uint4 wl[G][2], wh[G][2]; };  // weights only: X comes from L1 at compute time
  // thread t owns k in [8t, 8t+8) and [32+8t, 32+8t+8) of every 64-chunk (same permutation for W and X)
  auto load_group = [&](Buf& bf, int tile, int grp) {
    const int row0 = tile * ROWS + rg * 16;
    const bf16* wa = p.W + static_cast<long long>(min(row0 + g, p.N - 1)) * p.ldw;      // clamped rows are
    const bf16* wb = p.W + static_cast<long long>(min(row0 + g + 8, p.N - 1)) * p.ldw;  // masked in the epilogue
    const bool live = tile < ntiles;
#pragma unroll
    for (int u = 0; u < G; ++u) {
      const int c = c0 + grp * G + u;
      const int k0 = c * 64 + 8 * t, k1 = k0 + 32;
      const bool in = live && c < c1;
      const bool ok0 = in && k0 < p.K, ok1 = in && k1 < p.K;
      bf.wl[u][0] = ldg_stream(wa + k0, ok0); bf.wl[u][1] = ldg_stream(wa + k1, ok1);
      bf.wh[u][0] = ldg_stream(wb + k0, ok0); bf.wh[u][1] = ldg_stream(wb + k1, ok1);
    }
  };
  float acc[NT][4];
  auto compute_group = [&](const Buf& bf, int grp, bool first_tile) {
    uint4 xa[G][2], xb[G][2];
#pragma unroll
    for (int u = 0; u < G; ++u) {
      const int c = c0 + grp * G + u;
      const int k0 = c * 64 + 8 * t, k1 = k0 + 32;
      const bool in = c < c1;
      const bool ok0 = in && k0 < p.K, ok1 = in && k1 < p.K;
      xa[u][0] = ldg_cached(x0 + k0, ok0 && x0ok); xa[u][1] = ldg_cached(x0 + k1, ok1 && x0ok);
      if (NT == 2) { xb[u][0] = ldg_cached(x1 + k0, ok0 && x1ok); xb[u][1] = ldg_cached(x1 + k1, ok1 && x1ok); }
    }
#pragma unroll
    for (int u = 0; u < G; ++u) {
      const uint32_t al[8] = {bf.wl[u][0].x, bf.wl[u][0].y, bf.wl[u][0].z, bf.wl[u][0].w, bf.wl[u][1].x, bf.wl[u][1].y, bf.wl[u][1].z, bf.wl[u][1].w};
      const uint32_t ah[8] = {bf.wh[u][0].x, bf.wh[u][0].y, bf.wh[u][0].z, bf.wh[u][0].w, bf.wh[u][1].x, bf.wh[u][1].y, bf.wh[u][1].z, bf.wh[u][1].w};
      const uint32_t b0[8] = {xa[u][0].x, xa[u][0].y, xa[u][0].z, xa[u][0].w, xa[u][1].x, xa[u][1].y, xa[u][1].z, xa[u][1].w};
      uint32_t b1[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (NT == 2) {
        b1[0] = xb[u][0].x; b1[1] = xb[u][0].y; b1[2] = xb[u][0].z; b1[3] = xb[u][0].w;
        b1[4] = xb[u][1].x; b1[5] = xb[u][1].y; b1[6] = xb[u][1].z; b1[7] = xb[u][1].w;
      }
      if (do_rms && first_tile && rg == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float2 f = unpack_bf16(b0[j]);
          sq0 += f.x * f.x + f.y * f.y;
          if (NT == 2) { float2 h2 = unpack_bf16(b1[j]); sq1 += h2.x * h2.x + h2.y * h2.y; }
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        mma16816(acc[0], al[2 * j], ah[2 * j], al[2 * j + 1], ah[2 * j + 1], b0[2 * j], b0[2 * j + 1]);
        if (NT == 2) mma16816(acc[1], al[2 * j], ah[2 * j], al[2 * j + 1], ah[2 * j + 1], b1[2 * j], b1[2 * j + 1]);
      }
    }
  };

  Buf buf0, buf1;
  pdl_trigger();
  // weights never depend on the previous kernel: two groups are requested before the dependency wait, and
  // the pipeline stays two groups ahead of the MMAs from then on
  load_group(buf0, blockIdx.x, 0);
  load_group(buf1, blockIdx.x, 1);
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
#pragma unroll
    for (int i = 0; i < NT; ++i) {
      red[par][warp][g][i * 8 + 2 * t] = acc[i][0];
      red[par][warp][g][i * 8 + 2 * t + 1] = acc[i][1];
      red[par][warp][g + 8][i * 8 + 2 * t] = acc[i][2];
      red[par][warp][g + 8][i * 8 + 2 * t + 1] = acc[i][3];
    }
    if (do_rms && first) {
      sq0 += __shfl_xor_sync(0xffffffffu, sq0, 1); sq0 += __shfl_xor_sync(0xffffffffu, sq0, 2);
      if (NT == 2) { sq1 += __shfl_xor_sync(0xffffffffu, sq1, 1); sq1 += __shfl_xor_sync(0xffffffffu, sq1, 2); }
      if (t == 0) { red_sq[warp][g] = sq0; if (NT == 2) red_sq[warp][8 + g] = sq1; }
    }
    __syncthreads();
    if (do_rms && first) {
      if (threadIdx.x < NT * 8) {
        float ss = 0.f;
#pragma unroll
        for (int s2 = 0; s2 < KS; ++s2) ss += red_sq[s2 * RG][threadIdx.x];  // row-group-0 warps cover every k once
        rstd_s[threadIdx.x] = rsqrtf(ss / p.K + p.rms_eps);
      }
      __syncthreads();
    }
    // ---- epilogue: one thread per (token, output column of this tile)
    for (int item = threadIdx.x; item < p.M * out_cols; item += 256) {
      const int tok = item / out_cols, j = item % out_cols;
      const int fa = j, fb = j + 16;                       // packed GLU layout: [16 x a | 16 x b]
      const int na = tile * ROWS + fa;                      // accumulator column (weight row)
      const int oc = glu ? tile * (ROWS / 2) + j : na;
      if (oc >= n_out_total) continue;
      float va = 0.f, vb_ = 0.f;
#pragma unroll
      for (int s2 = 0; s2 < KS; ++s2) {
        va += red[par][s2 * RG + fa / 16][fa % 16][tok];
        if (glu) vb_ += red[par][s2 * RG + (fb / 16) % RG][fb % 16][tok];
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
      else r = gemv_act(va, p.act);
      if (p.residual) r = __bfloat162float(p.residual[tok * p.ldr + oc]) + p.alpha * r;
      else r *= p.alpha;
      if (p.out_fp32) reinterpret_cast<float*>(p.out)[tok * p.ldo + oc] = r;
      else reinterpret_cast<bf16*>(p.out)[tok * p.ldo + oc] = __float2bfloat16(r);
    }
    par ^= 1;
    first = false;
  }
}

}  // namespace vb

using namespace vb;

// internal entry used by vb200_gemm_bf16 (gemm.cu) for M <= 16
int vb_launch_gemv(const void* A, int64_t lda, const void* W, int64_t ldw, void* out, int64_t ldo, int64_t M,
                   int64_t N, int64_t K, const vb_epilogue* e, cudaStream_t stream) {
  GemvParams p;
  p.W = reinterpret_cast<const bf16*>(W); p.ldw = ldw;
  p.X = reinterpret_cast<const bf16*>(A); p.ldx = lda;
  p.out = out; p.ldo = ldo;
  p.M = static_cast<int>(M); p.N = static_cast<int>(N); p.K = static_cast<int>(K);
  p.bias = reinterpret_cast<const bf16*>(e->bias);
  p.rowbias = reinterpret_cast<const bf16*>(e->rowbias);
  p.rowbias_rows = e->rowbias_rows > 0 ? static_cast<int>(e->rowbias_rows) : 1;
  p.residual = reinterpret_cast<const bf16*>(e->residual); p.ldr = e->ldr;
  p.alpha = e->alpha; p.act = e->act; p.glu = e->glu; p.out_fp32 = e->out_fp32;
  p.rowscale = e->rowscale; p.rms_eps = e->rms_eps;
  const bool glu = e->glu != VB_GLU_NONE;
  // 32-row CTAs when the packed GLU layout requires it or when 16-row CTAs would exceed ~4 per SM
  const bool rows32 = glu || (N / 16 > 6LL * vb_num_sms());
  const unsigned tiles = static_cast<unsigned>((N + (rows32 ? 31 : 15)) / (rows32 ? 32 : 16));
  const unsigned cap = 2u * static_cast<unsigned>(vb_num_sms());  // persistent: 2 CTAs per SM
  const unsigned grid = tiles < cap ? tiles : cap;
  cudaError_t err;
  if (M <= 8) {
    if (rows32) err = vb_launch(gemv_bf16_kernel<32, 1>, dim3(grid), dim3(256), 0, stream, p);
    else err = vb_launch(gemv_bf16_kernel<16, 1>, dim3(grid), dim3(256), 0, stream, p);
  } else {
    if (rows32) err = vb_launch(gemv_bf16_kernel<32, 2>, dim3(grid), dim3(256), 0, stream, p);
    else err = vb_launch(gemv_bf16_kernel<16, 2>, dim3(grid), dim3(256), 0, stream, p);
  }
  if (err != cudaSuccess) { vb_set_last_error(err); return VB_ERR_CUDA; }
  return VB_OK;
}
