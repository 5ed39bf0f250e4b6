// vitron_b200 — softmax(QK^T * scale + mask) V without materialising the score matrix.
//
// flash_attn_kernel: 64 query rows per CTA (4 warps x 16 rows), 64-key blocks streamed through a
// 2-stage cp.async ring, online softmax in fp32 registers, bf16 tensor-core MMAs
// (mma.sync m16n8k16; the wgmma version of this kernel is attention_tc.cu).
// Generic element strides let it read q/k/v in place from fused QKV GEMM outputs.
//
// Replaces: HF LlamaAttention eager path (prefill; restated in vitron/train/
// llama_flash_attn_monkey_patch.py:30-66), HF CLIPAttention (languagebind/image/
// modeling_image.py:69), xformers memory_efficient_attention (i2vgen util.py:253-258, GLIGEN
// attention.py:176,247), SEEM multi_head_attention_forward (utils/attn.py:296-316).
//
// attn_short_kernel: one warp per (sequence, head) for S <= 32 (temporal attention over frames:
// modeling_video.py:105-127, i2vgen util.py:1061-1066) — pure HBM streaming.
#include "common.cuh"
#include "vitron_b200.h"

namespace vb {

struct AttnParams {
  const bf16* q; const bf16* k; const bf16* v; bf16* o;
  long long q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh;
  int B, H, Sq, Skv, hd;
  float scale_log2;  // scale * log2(e)
  int causal;
  const int32_t* kv_len;
  const uint8_t* mask;
  long long m_sb, m_sh, m_sq;
};

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  const uint32_t d = smem_u32(dst);
  const int bytes = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                          uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

constexpr int FA_BM = 64, FA_BN = 64, FA_THREADS = 128;

// load `rows` x HD tile (row-major, `row_stride` elements apart) into smem [64][HD+8]
template <int HD>
__device__ __forceinline__ void load_tile(bf16* s, const bf16* g, long long row_stride, int rows_valid, int hd) {
  constexpr int LD = HD + 8;
  constexpr int CH = HD / 8;
  for (int i = threadIdx.x; i < 64 * CH; i += FA_THREADS) {
    const int r = i / CH, c = (i % CH) * 8;
    const bool ok = (r < rows_valid) && (c < hd);
    const bf16* src = ok ? g + r * row_stride + c : g;
    cp_async16(s + r * LD + c, src, ok);
  }
}

template <int HD>
__global__ void __launch_bounds__(FA_THREADS) flash_attn_kernel(const AttnParams p) {
  constexpr int LD = HD + 8;       // padded row (elements): odd multiple of 16 B -> conflict-free ldmatrix
  constexpr int KS = HD / 16;      // k-steps over the head dim
  constexpr int NT = HD / 8;       // output n-tiles
  extern __shared__ __align__(16) uint8_t fa_smem[];
  bf16* sQ = reinterpret_cast<bf16*>(fa_smem);
  bf16* sK = sQ + 64 * LD;         // [2][64][LD]
  pdl_trigger();
  pdl_wait();
  bf16* sV = sK + 2 * 64 * LD;     // [2][64][LD]

  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int q0 = qb * FA_BM;
  const int kv_len = p.kv_len ? min(p.kv_len[b], p.Skv) : p.Skv;
  const int causal_off = p.Skv - p.Sq;  // key j visible to query i iff j <= i + (Skv - Sq)

  const bf16* qg = p.q + b * p.q_sb + h * p.q_sh + static_cast<long long>(q0) * p.q_ss;
  const bf16* kg = p.k + b * p.k_sb + h * p.k_sh;
  const bf16* vg = p.v + b * p.v_sb + h * p.v_sh;

  int kv_end = kv_len;
  if (p.causal) kv_end = min(kv_len, q0 + FA_BM + causal_off);
  const int nblk = kv_end > 0 ? (kv_end + FA_BN - 1) / FA_BN : 0;

  load_tile<HD>(sQ, qg, p.q_ss, p.Sq - q0, p.hd);
  if (nblk > 0) {
    load_tile<HD>(sK, kg, p.k_ss, kv_end, p.hd);
    load_tile<HD>(sV, vg, p.v_ss, kv_end, p.hd);
  }
  cp_async_commit();

  float o_acc[NT][4];
#pragma unroll
  for (int i = 0; i < NT; ++i) o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  uint32_t qf[KS][4];

  const int row_lo = q0 + warp * 16 + g;  // this thread's two query rows: row_lo, row_lo + 8
  const uint8_t* mrow0 = nullptr;
  const uint8_t* mrow1 = nullptr;
  if (p.mask) {
    const uint8_t* mb = p.mask + b * p.m_sb + h * p.m_sh;
    mrow0 = mb + static_cast<long long>(min(row_lo, p.Sq - 1)) * p.m_sq;
    mrow1 = mb + static_cast<long long>(min(row_lo + 8, p.Sq - 1)) * p.m_sq;
  }

  for (int j = 0; j < nblk; ++j) {
    cp_async_wait_all();
    __syncthreads();
    if (j == 0) {
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        const uint32_t a = smem_u32(sQ + (warp * 16 + (lane & 15)) * LD + ks * 16 + (lane >> 4) * 8);
        ldsm_x4(a, qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
      }
    }
    if (j + 1 < nblk) {
      const int k1 = (j + 1) * FA_BN;
      load_tile<HD>(sK + ((j + 1) & 1) * 64 * LD, kg + static_cast<long long>(k1) * p.k_ss, p.k_ss, kv_end - k1, p.hd);
      load_tile<HD>(sV + ((j + 1) & 1) * 64 * LD, vg + static_cast<long long>(k1) * p.v_ss, p.v_ss, kv_end - k1, p.hd);
      cp_async_commit();
    }
    const bf16* cK = sK + (j & 1) * 64 * LD;
    const bf16* cV = sV + (j & 1) * 64 * LD;

    // ---- S = Q K^T  (16 x 64 per warp)
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {  // pairs of 8-key tiles
        uint32_t b0, b1, b2, b3;
        const uint32_t a = smem_u32(cK + (np * 16 + (lane & 7) + (lane >> 4) * 8) * LD + ks * 16 + ((lane >> 3) & 1) * 8);
        ldsm_x4(a, b0, b1, b2, b3);
        mma_16816(s[2 * np], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], b0, b1);
        mma_16816(s[2 * np + 1], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], b2, b3);
      }
    }

    // ---- masking + online softmax
    const int kbase = j * FA_BN;
    const bool need_mask = (kbase + FA_BN > kv_end) || p.causal || (p.mask != nullptr);
    if (need_mask) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = kbase + nt * 8 + 2 * t + (e & 1);
          const int row = row_lo + (e >> 1) * 8;
          bool dead = key >= kv_end;
          if (p.causal && key > row + causal_off) dead = true;
          if (!dead && p.mask && row < p.Sq) dead = ((e >> 1) ? mrow1 : mrow0)[key] != 0;
          if (dead) s[nt][e] = -INFINITY;
        }
      }
    }
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float corr[2], moff[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      moff[r] = (mx[r] == -INFINITY) ? 0.f : mx[r] * p.scale_log2;
      corr[r] = (m_run[r] == -INFINITY) ? 0.f : exp2f(m_run[r] * p.scale_log2 - moff[r]);
      m_run[r] = mx[r];
      l_run[r] *= corr[r];
    }
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = exp2f(s[nt][0] * p.scale_log2 - moff[0]);
      s[nt][1] = exp2f(s[nt][1] * p.scale_log2 - moff[0]);
      s[nt][2] = exp2f(s[nt][2] * p.scale_log2 - moff[1]);
      s[nt][3] = exp2f(s[nt][3] * p.scale_log2 - moff[1]);
      rs[0] += s[nt][0] + s[nt][1];
      rs[1] += s[nt][2] + s[nt][3];
    }
    l_run[0] += rs[0];
    l_run[1] += rs[1];
#pragma unroll
    for (int i = 0; i < NT; ++i) {
      o_acc[i][0] *= corr[0]; o_acc[i][1] *= corr[0];
      o_acc[i][2] *= corr[1]; o_acc[i][3] *= corr[1];
    }

    // ---- O += P V
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // 16-key slices
      const uint32_t a0 = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
      const uint32_t a1 = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
      const uint32_t a2 = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      const uint32_t a3 = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int np = 0; np < NT / 2; ++np) {
        uint32_t b0, b1, b2, b3;
        const uint32_t a = smem_u32(cV + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + np * 16 + (lane >> 4) * 8);
        ldsm_x4_t(a, b0, b1, b2, b3);
        mma_16816(o_acc[2 * np], a0, a1, a2, a3, b0, b1);
        mma_16816(o_acc[2 * np + 1], a0, a1, a2, a3, b2, b3);
      }
    }
  }
  if (nblk == 0) {
    cp_async_wait_all();
    __syncthreads();
  }

  // ---- finalise: l across the quad, normalise, stage through smem (own rows of sQ), 16 B stores
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const float inv0 = l_run[0] > 0.f ? 1.f / l_run[0] : 0.f;
  const float inv1 = l_run[1] > 0.f ? 1.f / l_run[1] : 0.f;
  __syncwarp();
  bf16* so = sQ + warp * 16 * LD;
#pragma unroll
  for (int i = 0; i < NT; ++i) {
    *reinterpret_cast<uint32_t*>(so + g * LD + i * 8 + 2 * t) = pack_bf16(o_acc[i][0] * inv0, o_acc[i][1] * inv0);
    *reinterpret_cast<uint32_t*>(so + (g + 8) * LD + i * 8 + 2 * t) = pack_bf16(o_acc[i][2] * inv1, o_acc[i][3] * inv1);
  }
  __syncwarp();
  bf16* og = p.o + b * p.o_sb + h * p.o_sh;
  const int chunks = p.hd / 8;
  for (int i = lane; i < 16 * chunks; i += 32) {
    const int r = i / chunks, c = (i % chunks) * 8;
    const int row = q0 + warp * 16 + r;
    if (row < p.Sq)
      *reinterpret_cast<uint4*>(og + static_cast<long long>(row) * p.o_ss + c) = *reinterpret_cast<const uint4*>(so + r * LD + c);
  }
}

template <int HD>
static int launch_fa(const AttnParams& p, cudaStream_t stream) {
  constexpr int smem = 5 * 64 * (HD + 8) * 2;
  static bool attr = false;
  auto kern = flash_attn_kernel<HD>;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
    attr = true;
  }
  dim3 grid((p.Sq + FA_BM - 1) / FA_BM, p.H, p.B);
  { cudaError_t le = vb_launch(kern, grid, dim3(FA_THREADS), smem, stream, p); if (le != cudaSuccess) { vb_set_last_error(le); return VB_ERR_CUDA; } }
  VB_LAUNCH_CHECK();
  return VB_OK;
}

// ------------------------------------------------------------------ short sequences
struct ShortParams {
  const bf16* q; const bf16* k; const bf16* v; bf16* o;
  long long q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh;
  long long nseq; int H, S;
  long long inner;  // sequence index = outer * inner + in; offset = outer * *_so + in * *_sb
  long long q_so, k_so, v_so, o_so;
  float scale;
};

// one warp per (sequence, head); head_dim 64; S <= MAXS
template <int MAXS, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) attn_short_kernel(const ShortParams p) {
  constexpr int HD = 64;
  __shared__ __align__(16) bf16 sq[WARPS][MAXS][HD + 2];
  __shared__ __align__(16) bf16 sk[WARPS][MAXS][HD + 2];
  __shared__ __align__(16) bf16 sv[WARPS][MAXS][HD + 2];
  __shared__ float sp[WARPS][MAXS][MAXS + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long item = static_cast<long long>(blockIdx.x) * WARPS + warp;
  if (item >= p.nseq * p.H) return;
  const long long seq = item / p.H;
  const int h = static_cast<int>(item % p.H);
  const long long so = seq / p.inner, si = seq % p.inner;
  const bf16* qg = p.q + so * p.q_so + si * p.q_sb + h * p.q_sh;
  const bf16* kg = p.k + so * p.k_so + si * p.k_sb + h * p.k_sh;
  const bf16* vg = p.v + so * p.v_so + si * p.v_sb + h * p.v_sh;
  const int S = p.S;
  // each lane moves 4 bytes; a row of 64 bf16 = 32 lanes x 2 elements (fully coalesced 128 B)
  for (int s = 0; s < S; ++s) {
    *reinterpret_cast<uint32_t*>(&sq[warp][s][lane * 2]) = *reinterpret_cast<const uint32_t*>(qg + s * p.q_ss + lane * 2);
    *reinterpret_cast<uint32_t*>(&sk[warp][s][lane * 2]) = *reinterpret_cast<const uint32_t*>(kg + s * p.k_ss + lane * 2);
    *reinterpret_cast<uint32_t*>(&sv[warp][s][lane * 2]) = *reinterpret_cast<const uint32_t*>(vg + s * p.v_ss + lane * 2);
  }
  __syncwarp();
  for (int idx = lane; idx < S * S; idx += 32) {
    const int i = idx / S, j = idx % S;
    float acc = 0.f;
#pragma unroll 16
    for (int d = 0; d < HD; d += 2) {
      float2 a = __bfloat1622float2(*reinterpret_cast<const bf162*>(&sq[warp][i][d]));
      float2 b = __bfloat1622float2(*reinterpret_cast<const bf162*>(&sk[warp][j][d]));
      acc += a.x * b.x + a.y * b.y;
    }
    sp[warp][i][j] = acc * p.scale;
  }
  __syncwarp();
  if (lane < S) {
    float m = -INFINITY;
    for (int j = 0; j < S; ++j) m = fmaxf(m, sp[warp][lane][j]);
    float l = 0.f;
    for (int j = 0; j < S; ++j) { float e = __expf(sp[warp][lane][j] - m); sp[warp][lane][j] = e; l += e; }
    const float inv = 1.f / l;
    for (int j = 0; j < S; ++j) sp[warp][lane][j] *= inv;
  }
  __syncwarp();
  bf16* og = p.o + so * p.o_so + si * p.o_sb + h * p.o_sh;
  for (int i = 0; i < S; ++i) {
    float a0 = 0.f, a1 = 0.f;
    for (int j = 0; j < S; ++j) {
      const float pj = sp[warp][i][j];
      float2 vv = __bfloat1622float2(*reinterpret_cast<const bf162*>(&sv[warp][j][lane * 2]));
      a0 += pj * vv.x;
      a1 += pj * vv.y;
    }
    *reinterpret_cast<uint32_t*>(og + i * p.o_ss + lane * 2) = pack_bf16(a0, a1);
  }
}

// S <= 16, head_dim 64, 16-byte aligned rows: one warp per (sequence, head) on mma.sync tensor cores.
// The three 16 x 64 operand tiles arrive with twelve independent 16-byte loads per lane (rows >= S are
// zero-filled), go through warp-private shared memory for ldmatrix, and the whole attention is
// 8 (QK^T) + 8 (PV) m16n8k16 MMAs; the result leaves through the Q tile with 16-byte stores.
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) attn_short_mma_kernel(const ShortParams p) {
  constexpr int HD = 64, LD = HD + 8;
  __shared__ __align__(16) bf16 sm[WARPS][3][16][LD];
  pdl_trigger();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long item = static_cast<long long>(blockIdx.x) * WARPS + warp;
  if (item >= p.nseq * p.H) return;  // no CTA-wide barriers below
  const long long seq = item / p.H;
  const int h = static_cast<int>(item % p.H);
  const long long so = seq / p.inner, si = seq % p.inner;
  const bf16* qg = p.q + so * p.q_so + si * p.q_sb + h * p.q_sh;
  const bf16* kg = p.k + so * p.k_so + si * p.k_sb + h * p.k_sh;
  const bf16* vg = p.v + so * p.v_so + si * p.v_sb + h * p.v_sh;
  const int S = p.S;
  const int piece = (lane & 7) * 8, r0 = lane >> 3;
  uint4 rq[4], rk[4], rv[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = r0 + 4 * i;
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    rq[i] = rk[i] = rv[i] = z;
    if (row < S) {
      rq[i] = __ldg(reinterpret_cast<const uint4*>(qg + row * p.q_ss + piece));
      rk[i] = __ldg(reinterpret_cast<const uint4*>(kg + row * p.k_ss + piece));
      rv[i] = __ldg(reinterpret_cast<const uint4*>(vg + row * p.v_ss + piece));
    }
  }
  bf16 (*sq)[LD] = sm[warp][0];
  bf16 (*sk)[LD] = sm[warp][1];
  bf16 (*sv)[LD] = sm[warp][2];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = r0 + 4 * i;
    *reinterpret_cast<uint4*>(&sq[row][piece]) = rq[i];
    *reinterpret_cast<uint4*>(&sk[row][piece]) = rk[i];
    *reinterpret_cast<uint4*>(&sv[row][piece]) = rv[i];
  }
  __syncwarp();
  const int g = lane >> 2, t = lane & 3;
  float sc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
    ldsm_x4(smem_u32(&sq[lane & 15][ks * 16 + (lane >> 4) * 8]), a0, a1, a2, a3);
    ldsm_x4(smem_u32(&sk[(lane & 7) + (lane >> 4) * 8][ks * 16 + ((lane >> 3) & 1) * 8]), b0, b1, b2, b3);
    mma_16816(sc[0], a0, a1, a2, a3, b0, b1);
    mma_16816(sc[1], a0, a1, a2, a3, b2, b3);
  }
  // softmax over the S valid keys; thread holds rows g (e = 0, 1) and g + 8 (e = 2, 3), keys nt * 8 + 2t + (e & 1)
  const float sl2 = p.scale * 1.4426950408889634f;
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (nt * 8 + 2 * t + (e & 1) >= S) sc[nt][e] = -INFINITY;
      mx[e >> 1] = fmaxf(mx[e >> 1], sc[nt][e]);
    }
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
  }
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      sc[nt][e] = exp2f((sc[nt][e] - mx[e >> 1]) * sl2);
      sum[e >> 1] += sc[nt][e];
    }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
    sum[r] = 1.f / sum[r];
  }
  const uint32_t pa0 = pack_bf16(sc[0][0] * sum[0], sc[0][1] * sum[0]);
  const uint32_t pa1 = pack_bf16(sc[0][2] * sum[1], sc[0][3] * sum[1]);
  const uint32_t pa2 = pack_bf16(sc[1][0] * sum[0], sc[1][1] * sum[0]);
  const uint32_t pa3 = pack_bf16(sc[1][2] * sum[1], sc[1][3] * sum[1]);
  float oa[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) oa[i][0] = oa[i][1] = oa[i][2] = oa[i][3] = 0.f;
#pragma unroll
  for (int np = 0; np < 4; ++np) {
    uint32_t b0, b1, b2, b3;
    ldsm_x4_t(smem_u32(&sv[(lane & 7) + ((lane >> 3) & 1) * 8][np * 16 + (lane >> 4) * 8]), b0, b1, b2, b3);
    mma_16816(oa[2 * np], pa0, pa1, pa2, pa3, b0, b1);
    mma_16816(oa[2 * np + 1], pa0, pa1, pa2, pa3, b2, b3);
  }
  // O through the (already consumed) Q tile, then 16-byte row pieces
  __syncwarp();
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    *reinterpret_cast<uint32_t*>(&sq[g][nt * 8 + 2 * t]) = pack_bf16(oa[nt][0], oa[nt][1]);
    *reinterpret_cast<uint32_t*>(&sq[g + 8][nt * 8 + 2 * t]) = pack_bf16(oa[nt][2], oa[nt][3]);
  }
  __syncwarp();
  bf16* og = p.o + so * p.o_so + si * p.o_sb + h * p.o_sh;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = r0 + 4 * i;
    if (row < S) *reinterpret_cast<uint4*>(og + row * p.o_ss + piece) = *reinterpret_cast<const uint4*>(&sq[row][piece]);
  }
}

}  // namespace vb

using namespace vb;

int vb_attention_tc(const void* q, const void* k, const void* v, void* out, int64_t B, int64_t H, int64_t Sq,
                    int64_t Skv, int64_t head_dim, int64_t q_sb, int64_t q_ss, int64_t q_sh, int64_t k_sb,
                    int64_t k_ss, int64_t k_sh, int64_t v_sb, int64_t v_ss, int64_t v_sh, int64_t o_sb, int64_t o_ss,
                    int64_t o_sh, float scale, int causal, const int32_t* kv_len, const uint8_t* mask, int64_t m_sb,
                    int64_t m_sh, int64_t m_sq, void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t vb_attention_tc_workspace(int64_t B, int64_t H, int64_t Sq, int64_t Skv, int64_t head_dim, int causal);

static int g_attention_impl = 0;  // 0 auto, 1 mma.sync only, 2 wgmma whenever the shape is supported
extern "C" int vb200_set_attention_impl(int impl) {
  VB_CHECK_ARG(impl >= 0 && impl <= 2);
  g_attention_impl = impl;
  return VB_OK;
}

extern "C" size_t vb200_attention_workspace_size(int64_t B, int64_t H, int64_t Sq, int64_t Skv, int64_t head_dim, int causal) {
  if (B <= 0 || H <= 0 || Sq <= 0 || Skv <= 0 || head_dim <= 0) return 0;
  if (Sq < 96 && g_attention_impl != 2) return 0;
  return vb_attention_tc_workspace(B, H, Sq, Skv, head_dim, causal);
}

extern "C" int vb200_attention(const void* q, const void* k, const void* v, void* out, int64_t B,
                               int64_t H, int64_t Sq, int64_t Skv, int64_t head_dim, int64_t q_sb,
                               int64_t q_ss, int64_t q_sh, int64_t k_sb, int64_t k_ss, int64_t k_sh,
                               int64_t v_sb, int64_t v_ss, int64_t v_sh, int64_t o_sb, int64_t o_ss,
                               int64_t o_sh, float scale, int causal, const int32_t* kv_len,
                               const uint8_t* mask, int64_t m_sb, int64_t m_sh, int64_t m_sq,
                               cudaStream_t stream) {
  return vb200_attention_ws(q, k, v, out, B, H, Sq, Skv, head_dim, q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb,
                            o_ss, o_sh, scale, causal, kv_len, mask, m_sb, m_sh, m_sq, nullptr, 0, stream);
}

extern "C" int vb200_attention_ws(const void* q, const void* k, const void* v, void* out, int64_t B,
                                  int64_t H, int64_t Sq, int64_t Skv, int64_t head_dim, int64_t q_sb,
                                  int64_t q_ss, int64_t q_sh, int64_t k_sb, int64_t k_ss, int64_t k_sh,
                                  int64_t v_sb, int64_t v_ss, int64_t v_sh, int64_t o_sb, int64_t o_ss,
                                  int64_t o_sh, float scale, int causal, const int32_t* kv_len,
                                  const uint8_t* mask, int64_t m_sb, int64_t m_sh, int64_t m_sq,
                                  void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  VB_CHECK_ARG(q && k && v && out);
  VB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Skv >= 0 && head_dim > 0 && head_dim % 8 == 0);
  VB_CHECK_ARG(H <= 65535 && B <= 65535);
  const int64_t strides[12] = {q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh};
  for (int i = 0; i < 12; ++i) VB_CHECK_ARG(strides[i] % 8 == 0);
  // wgmma kernel (attention_tc.cu): head_dim 64 / 128 natively, 40 / 80 / 160 zero-padded by the TMA unit,
  // boolean masks applied in registers; taken whenever the query rows fill most of a 128-row tile. Short queries and
  // operand layouts a tensor map cannot describe stay on the mma.sync kernel below.
  if (g_attention_impl != 1 && Skv >= 1 && (Sq >= 96 || g_attention_impl == 2)) {
    int r = vb_attention_tc(q, k, v, out, B, H, Sq, Skv, head_dim, q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss,
                            v_sh, o_sb, o_ss, o_sh, scale, causal, kv_len, mask, m_sb, m_sh, m_sq, workspace, workspace_bytes, stream);
    if (r != VB_ERR_UNSUPPORTED) return r;
  }
  AttnParams p;
  p.q = reinterpret_cast<const bf16*>(q); p.k = reinterpret_cast<const bf16*>(k);
  p.v = reinterpret_cast<const bf16*>(v); p.o = reinterpret_cast<bf16*>(out);
  p.q_sb = q_sb; p.q_ss = q_ss; p.q_sh = q_sh; p.k_sb = k_sb; p.k_ss = k_ss; p.k_sh = k_sh;
  p.v_sb = v_sb; p.v_ss = v_ss; p.v_sh = v_sh; p.o_sb = o_sb; p.o_ss = o_ss; p.o_sh = o_sh;
  p.B = (int)B; p.H = (int)H; p.Sq = (int)Sq; p.Skv = (int)Skv; p.hd = (int)head_dim;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.causal = causal; p.kv_len = kv_len; p.mask = mask; p.m_sb = m_sb; p.m_sh = m_sh; p.m_sq = m_sq;
  if (head_dim <= 48) return launch_fa<48>(p, stream);
  if (head_dim <= 64) return launch_fa<64>(p, stream);
  if (head_dim <= 80) return launch_fa<80>(p, stream);
  if (head_dim <= 128) return launch_fa<128>(p, stream);
  if (head_dim <= 160) return launch_fa<160>(p, stream);
  return VB_ERR_UNSUPPORTED;
}

extern "C" int vb200_attention_short(const void* q, const void* k, const void* v, void* out,
                                     int64_t nseq, int64_t H, int64_t S, int64_t head_dim,
                                     int64_t q_sb, int64_t q_ss, int64_t q_sh, int64_t k_sb,
                                     int64_t k_ss, int64_t k_sh, int64_t v_sb, int64_t v_ss,
                                     int64_t v_sh, int64_t o_sb, int64_t o_ss, int64_t o_sh,
                                     int64_t inner, int64_t q_so, int64_t k_so, int64_t v_so,
                                     int64_t o_so, float scale, cudaStream_t stream) {
  VB_CHECK_ARG(q && k && v && out);
  VB_CHECK_ARG(nseq > 0 && H > 0 && S > 0 && S <= 32 && head_dim == 64);
  if (inner <= 0) { inner = nseq; q_so = k_so = v_so = o_so = 0; }
  VB_CHECK_ARG(q_so % 2 == 0 && k_so % 2 == 0 && v_so % 2 == 0 && o_so % 2 == 0);
  const int64_t strides[12] = {q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh};
  for (int i = 0; i < 12; ++i) VB_CHECK_ARG(strides[i] % 2 == 0);
  ShortParams p;
  p.q = reinterpret_cast<const bf16*>(q); p.k = reinterpret_cast<const bf16*>(k);
  p.v = reinterpret_cast<const bf16*>(v); p.o = reinterpret_cast<bf16*>(out);
  p.q_sb = q_sb; p.q_ss = q_ss; p.q_sh = q_sh; p.k_sb = k_sb; p.k_ss = k_ss; p.k_sh = k_sh;
  p.v_sb = v_sb; p.v_ss = v_ss; p.v_sh = v_sh; p.o_sb = o_sb; p.o_ss = o_ss; p.o_sh = o_sh;
  p.nseq = nseq; p.H = (int)H; p.S = (int)S; p.scale = scale;
  p.inner = inner; p.q_so = q_so; p.k_so = k_so; p.v_so = v_so; p.o_so = o_so;
  const long long items = nseq * H;
  // tensor-core kernel when every row piece can move as 16 bytes
  bool vec16 = S <= 16 && ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                            reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  const int64_t all[16] = {q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh, q_so, k_so, v_so, o_so};
  for (int i = 0; i < 16; ++i) vec16 = vec16 && (all[i] % 8 == 0);
  if (vec16) {
    { cudaError_t le = vb_launch(attn_short_mma_kernel<4>, dim3(static_cast<unsigned>((items + 3) / 4)), dim3(128), 0, stream, p); if (le != cudaSuccess) { vb_set_last_error(le); return VB_ERR_CUDA; } }
    VB_LAUNCH_CHECK();
    return VB_OK;
  }
  if (S <= 8) attn_short_kernel<8, 4><<<static_cast<unsigned>((items + 3) / 4), 128, 0, stream>>>(p);
  else if (S <= 16) attn_short_kernel<16, 4><<<static_cast<unsigned>((items + 3) / 4), 128, 0, stream>>>(p);
  else attn_short_kernel<32, 2><<<static_cast<unsigned>((items + 1) / 2), 64, 0, stream>>>(p);
  VB_LAUNCH_CHECK();
  return VB_OK;
}
