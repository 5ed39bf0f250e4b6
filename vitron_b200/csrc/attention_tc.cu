// vitron_b200 — flash attention on sm_90a warpgroup MMA (wgmma), operands fed by TMA through mbarriers.
//
//   O = softmax(Q K^T * scale [causal, kv_len, bool mask]) V     bf16 in / out, fp32 math
//   head_dim 64 / 128 natively; 40 / 80 / 160 (GLIGEN, attention.py:192-257) run the 64 / 128 / 192-column
//   instantiation: the tensor maps carry the true head_dim, so the TMA unit zero-fills the padding columns of
//   Q / K / V in shared memory (they add 0 to QK^T and produce zero O columns that are never stored).
//   Boolean masks (SEEM masked cross-attention, utils/attn.py:296-316): uint8 [B|1, H|1, Sq, Skv], non-zero = masked
//   out, applied to S in registers; a row with every key masked yields zeros.
//
// One CTA = 128 query rows of one (batch, head); keys stream through in blocks of 64.
//   warpgroup 0      TMA producer (one thread): Q once, K_j / V_j into 2-stage 128B-swizzled rings (4-D tensor maps
//                    over the caller's strided [B, S, H, D] views, so fused QKV buffers are read in place)
//   warpgroups 1, 2  query rows [64 (wg - 1), +64): S_j = Q K_j^T (wgmma m64 n64, both operands K-major in shared
//                    memory) into registers, online softmax in registers (a row lives in the 4 threads of a quad), then
//                    O += P_j V_j with P_j as the register A operand (the S accumulator fragment IS the A fragment
//                    layout, so P never touches shared memory) and V_j read MN-major (transposed B descriptor).
// setmaxnreg hands the producer's registers to the consumers (O of a 64 x 192 tile is 96 fp32 per thread).
//
// Replaces (when there is no boolean mask and D in {64, 128}) the mma.sync kernel of attention.cu for:
// LLaMA prefill, CLIP ViT, UNet spatial self/cross attention, SEEM pixel-decoder encoder, SEEM self-attn.
#include "common.cuh"
#include "vitron_b200.h"
#include "wgmma.cuh"

#include <type_traits>

namespace vb {

constexpr int TC_BM = 128;  // query rows per CTA
constexpr int TC_BN = 64;   // keys per block
constexpr int TC_THREADS = 384;  // producer warpgroup + two consumer warpgroups

struct TcAttnParams {
  bf16* o;
  long long o_sb, o_ss, o_sh;
  int B, H, Sq, Skv;
  int D;                 // true head dim (<= the kernel's HD; the difference is zero padding)
  float scale_log2;
  int causal;
  const int32_t* kv_len;
  const uint8_t* mask;   // or null
  long long m_sb, m_sh, m_sq;
  int splits;            // > 1: the key blocks are divided over `splits` CTAs per query tile (few-query attention: SEEM's
  float* ws_o;           //      101 queries over 16384 keys would otherwise run on 8 CTAs); each writes its un-normalised
  float* ws_ml;          //      O (fp32) and (m, l) to the workspace, attn_split_merge_kernel combines them
};

// Paged instantiation (vb200_attention_paged): K / V come from a paged cache [num_pages, H, 64, 128] through the block
// table, one 64-key block = one (page, head) box. Row b holds q_len[b] queries at cache positions q_start[b] + i;
// query i sees key j iff j <= q_start[b] + i (causal, kv_len and mask of the base struct are unused).
struct TcPagedParams : TcAttnParams {
  const int32_t* block_table;   // [B, max_pages]
  int max_pages;
  const int32_t* q_start;       // [B]
  const int32_t* q_len;         // [B]
  int max_kv_len;               // keys at positions >= max_kv_len are never read
};

// Bounded mbarrier wait: a protocol or descriptor bug must never hang the GPU. After 4 s without progress the
// waiter records (site id, block) in g_tc_watchdog and TRAPS: the launch fails with a sticky CUDA error that the
// next vb200_* call / stream synchronisation reports (VB_ERR_CUDA) — a timed-out attention never returns garbage
// as if it were a result. The abort flag only short-cuts the other waiters of the CTA until the trap lands.
__device__ unsigned int g_tc_watchdog[4];

__device__ __forceinline__ unsigned long long gtime_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ void tc_wait_slow(uint64_t* bar, uint32_t parity, volatile uint32_t* abort_flag, int site) {
  const unsigned long long t0 = gtime_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (*abort_flag) return;
    if (gtime_ns() - t0 > 4000000000ull) {
      *abort_flag = 1;
      if (atomicCAS(&g_tc_watchdog[0], 0u, static_cast<unsigned int>(site)) == 0u) {
        g_tc_watchdog[1] = blockIdx.x | (blockIdx.y << 12) | (blockIdx.z << 22);
        g_tc_watchdog[2] = threadIdx.x;
      }
      __threadfence_system();
      __trap();
    }
  }
}

__device__ __forceinline__ void tc_wait(uint64_t* bar, uint32_t parity, volatile uint32_t* abort_flag, int site) {
#pragma unroll 1
  for (int i = 0; i < 64; ++i)
    if (mbar_try_wait(bar, parity)) return;
  tc_wait_slow(bar, parity, abort_flag, site);
}

__device__ __forceinline__ float ex2_approx(float x) {  // MUFU.EX2, flush-to-zero: exp2(-inf) = 0, no denormal fix-up
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int HD>
constexpr int tc_smem_bytes() {
  return TC_BM * HD * 2 + 4 * TC_BN * HD * 2 + 128;   // Q + 2-stage K and V rings + barriers
}

template <int HD, typename P>
__global__ void __launch_bounds__(TC_THREADS, 1)
flash_attn_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                     const __grid_constant__ CUtensorMap tmap_v, const P p) {
  constexpr bool PAGED = std::is_same<P, TcPagedParams>::value;
  pdl_trigger();
  pdl_wait();   // (the mbarrier set-up below touches no global data, but the kernel's first TMA load follows at once)
  constexpr int KC = HD / 64;                   // 64-element chunks along the head dim
  constexpr int Q_BYTES = TC_BM * HD * 2;       // [KC][128 rows][64]   K-major
  constexpr int K_BYTES = TC_BN * HD * 2;       // [KC][64 keys][64]    K-major
  constexpr int V_BYTES = TC_BN * HD * 2;       // [KC][64 keys][64]    read MN-major by the P V product

  // No static shared memory in this kernel, so the dynamic window starts at the (1024-byte aligned) base of the
  // CTA's allocation, as the 128B swizzle atoms require.
  extern __shared__ __align__(1024) uint8_t smem[];
  if (smem_u32(smem) & 1023u) __trap();
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Q_BYTES;          // 2 stages
  uint8_t* sV = sK + 2 * K_BYTES;      // 2 stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * V_BYTES);
  uint64_t* q_full = bars;             // 1
  uint64_t* k_full = bars + 1;         // 2
  uint64_t* k_empty = bars + 3;        // 2 (one arrival per consumer warp: wgmma.wait_group completes per warp)
  uint64_t* v_full = bars + 5;         // 2
  uint64_t* v_empty = bars + 7;        // 2 (one arrival per consumer warp)
  volatile uint32_t* abort_flag = reinterpret_cast<volatile uint32_t*>(bars + 9);

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int qb = blockIdx.x / p.splits, sp = blockIdx.x - qb * p.splits, h = blockIdx.y, b = blockIdx.z;
  const int q0 = qb * TC_BM;
  int causal_off, kv_end;
  int q_valid = p.Sq;   // query rows at or past it are written as zeros (paged: q_len[b])
  if constexpr (PAGED) {
    const int qs = max(p.q_start[b], 0);
    q_valid = max(0, min(p.q_len[b], p.Sq));
    causal_off = qs;
    kv_end = q0 < q_valid ? min(qs + min(q0 + TC_BM, q_valid), p.max_kv_len) : 0;
  } else {
    const int kv_len = p.kv_len ? min(p.kv_len[b], p.Skv) : p.Skv;
    causal_off = p.Skv - p.Sq;
    kv_end = kv_len;
    if (p.causal) kv_end = min(kv_len, q0 + TC_BM + causal_off);
  }
  const int nblk_all = kv_end > 0 ? (kv_end + TC_BN - 1) / TC_BN : 0;
  // this CTA's share of the key blocks: [jb0, jb0 + nblk)
  const int per_split = (nblk_all + p.splits - 1) / p.splits;
  const int jb0 = sp * per_split;
  const int nblk = max(0, min(nblk_all, jb0 + per_split) - jb0);

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_q);
    prefetch_tmap(&tmap_k);
    prefetch_tmap(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], 8);
      mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], 8);
    }
    *abort_flag = 0;
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================================================== TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (tid == 0 && nblk > 0) {
      mbar_arrive_expect_tx(q_full, Q_BYTES);
#pragma unroll
      for (int c = 0; c < KC; ++c) tma_load_4d(sQ + c * (TC_BM * 128), &tmap_q, q_full, c * 64, q0, h, b);
      // paged: key block (jb0 + j) is the (page, head) box of the row's (jb0 + j)-th page; the id of the next block's page
      // is loaded one iteration ahead, so its global-load latency overlaps the wait for a free ring slot
      const int32_t* pages = nullptr;
      int next_page = 0;
      if constexpr (PAGED) {
        pages = p.block_table + static_cast<long long>(b) * p.max_pages + jb0;
        next_page = pages[0];
      }
      for (int j = 0; j < nblk; ++j) {
        const int st = j & 1;
        const uint32_t ph = (j >> 1) & 1;
        int page = 0;
        if constexpr (PAGED) {
          page = next_page;
          if (j + 1 < nblk) next_page = pages[j + 1];
        }
        tc_wait(&k_empty[st], ph ^ 1, abort_flag, 5);
        mbar_arrive_expect_tx(&k_full[st], K_BYTES);
        if constexpr (PAGED) {
#pragma unroll
          for (int c = 0; c < KC; ++c) tma_load_4d(sK + st * K_BYTES + c * (TC_BN * 128), &tmap_k, &k_full[st], c * 64, 0, h, page);
        } else {
#pragma unroll
          for (int c = 0; c < KC; ++c) tma_load_4d(sK + st * K_BYTES + c * (TC_BN * 128), &tmap_k, &k_full[st], c * 64, (jb0 + j) * TC_BN, h, b);
        }
        tc_wait(&v_empty[st], ph ^ 1, abort_flag, 6);
        mbar_arrive_expect_tx(&v_full[st], V_BYTES);
        if constexpr (PAGED) {
#pragma unroll
          for (int c = 0; c < KC; ++c) tma_load_4d(sV + st * V_BYTES + c * (TC_BN * 128), &tmap_v, &v_full[st], c * 64, 0, h, page);
        } else {
#pragma unroll
          for (int c = 0; c < KC; ++c) tma_load_4d(sV + st * V_BYTES + c * (TC_BN * 128), &tmap_v, &v_full[st], c * 64, (jb0 + j) * TC_BN, h, b);
        }
      }
    }
    return;
  }

  // ===================================================== consumers: QK^T, softmax, PV, epilogue
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cwg = wg - 1;
  const int lane = tid & 31;
  // fragment rows of this thread: tile rows r_lo (h = 0) and r_lo + 8 (h = 1); columns 8i + cq + {0, 1}
  const int r_lo = cwg * 64 + (tid >> 5) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};   // running row max (score units)
  float l_part[2] = {0.f, 0.f};              // this thread's share of the row sums (quad-reduced at the end)
  const uint8_t* mrow[2] = {nullptr, nullptr};
  if (!PAGED && p.mask != nullptr) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int qrow = q0 + r_lo + 8 * hh;
      if (qrow < p.Sq) mrow[hh] = p.mask + b * p.m_sb + h * p.m_sh + static_cast<long long>(qrow) * p.m_sq;
    }
  }
  if (nblk > 0) tc_wait(q_full, 0, abort_flag, 1);
  for (int j = 0; j < nblk; ++j) {
    const int st = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    // ---- S = Q K_j^T
    float s[TC_BN / 2];
    tc_wait(&k_full[st], ph, abort_flag, 2);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      const uint32_t qa = smem_u32(sQ) + (ks / 4) * (TC_BM * 128) + cwg * (64 * 128) + (ks % 4) * 32;
      const uint32_t ka = smem_u32(sK) + st * K_BYTES + (ks / 4) * (TC_BN * 128) + (ks % 4) * 32;
      Wgmma<TC_BN>::ss(s, gmma_desc_kmajor(qa), gmma_desc_kmajor(ka), ks > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(s);
    if (lane == 0) mbar_arrive(&k_empty[st]);

    // ---- masks: key range (kv_len, causal) and the boolean mask
    const int kbase = (jb0 + j) * TC_BN;
    const bool need_mask = (kbase + TC_BN > kv_end) || (p.causal && kbase + TC_BN - 1 > q0 + causal_off);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int qrow = q0 + r_lo + 8 * hh;
      if (need_mask) {
        const int lim = min(kv_end, p.causal ? qrow + causal_off + 1 : kv_end) - kbase;  // keys [0, lim) are live
#pragma unroll
        for (int i = 0; i < TC_BN / 8; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (8 * i + cq + e >= lim) s[4 * i + 2 * hh + e] = -INFINITY;
      }
      if (mrow[hh] != nullptr) {
#pragma unroll
        for (int i = 0; i < TC_BN / 8; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int kk = kbase + 8 * i + cq + e;
            if (kk < p.Skv && mrow[hh][kk]) s[4 * i + 2 * hh + e] = -INFINITY;
          }
      }
    }

    // ---- online softmax (exp2 domain), rows reduced over the 4 threads of a quad
    uint32_t pa[TC_BN / 16][4];   // P_j as bf16 A fragments, one per 16 keys
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < TC_BN / 8; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * hh], s[4 * i + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hh], mx);
      const float corr = m_run[hh] == -INFINITY ? 1.f : ex2_approx((m_run[hh] - m_new) * p.scale_log2);
      m_run[hh] = m_new;
      const float moff = m_new == -INFINITY ? 0.f : m_new * p.scale_log2;
      float ps = 0.f;
#pragma unroll
      for (int i = 0; i < TC_BN / 8; ++i) {
        const float p0 = ex2_approx(fmaf(s[4 * i + 2 * hh], p.scale_log2, -moff));
        const float p1 = ex2_approx(fmaf(s[4 * i + 2 * hh + 1], p.scale_log2, -moff));
        ps += p0 + p1;
        pa[i / 2][(i & 1) * 2 + hh] = pack_bf16(p0, p1);
      }
      l_part[hh] = l_part[hh] * corr + ps;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) {
        o[4 * i + 2 * hh] *= corr;
        o[4 * i + 2 * hh + 1] *= corr;
      }
    }

    // ---- O += P_j V_j
    tc_wait(&v_full[st], ph, abort_flag, 4);
    wgmma_fence_operand(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < TC_BN / 16; ++kk) {
      const uint32_t va = smem_u32(sV) + st * V_BYTES + kk * (16 * 128);   // +16 key rows
      Wgmma<HD>::rs_tb(o, pa[kk], gmma_desc_sw128(va, TC_BN * 128, 1024), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(o);
    if (lane == 0) mbar_arrive(&v_empty[st]);
  }

  // ---- epilogue: O / l -> bf16 -> global (or the un-normalised partial of this key range)
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_part[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int qrow = q0 + r_lo + 8 * hh;
    if (qrow >= p.Sq) continue;
    if (PAGED && qrow >= q_valid) {   // padding query of a shorter row: zeros (split: an empty partial)
      l = 0.f;
      m_run[hh] = -INFINITY;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) o[4 * i + 2 * hh] = o[4 * i + 2 * hh + 1] = 0.f;
    }
    if (p.splits > 1) {
      const long long slot = ((static_cast<long long>(b) * p.H + h) * p.splits + sp) * p.Sq + qrow;
      if ((lane & 3) == 0) {
        p.ws_ml[slot * 2] = m_run[hh] == -INFINITY ? -INFINITY : m_run[hh] * p.scale_log2;
        p.ws_ml[slot * 2 + 1] = l;
      }
      float* orow_ws = p.ws_o + slot * HD;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i)
        if (8 * i + cq < p.D) *reinterpret_cast<float2*>(orow_ws + 8 * i + cq) = make_float2(o[4 * i + 2 * hh], o[4 * i + 2 * hh + 1]);
    } else {
      const float inv = l > 0.f ? 1.f / l : 0.f;
      bf16* orow = p.o + b * p.o_sb + h * p.o_sh + static_cast<long long>(qrow) * p.o_ss;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i)
        if (8 * i + cq < p.D)
          *reinterpret_cast<uint32_t*>(orow + 8 * i + cq) = pack_bf16(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
    }
  }
}

// out[b, q, h, :] = sum_s O_s 2^(m_s - M) / sum_s l_s 2^(m_s - M): one thread per 4 head-dim columns of a (b, h, q) row
__global__ void attn_split_merge_kernel(const float* __restrict__ ws_o, const float* __restrict__ ws_ml, bf16* __restrict__ out,
                                        long long o_sb, long long o_ss, long long o_sh, int B, int H, int Sq, int D, int HD, int splits) {
  pdl_trigger();
  pdl_wait();
  const int vecs = D / 4;
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(B) * H * Sq * vecs) return;
  const int v = static_cast<int>(idx % vecs);
  const long long row = idx / vecs;          // (b * H + h) * Sq + q
  const int q = static_cast<int>(row % Sq);
  const long long bh = row / Sq;
  float M = -INFINITY;
  for (int s = 0; s < splits; ++s) M = fmaxf(M, ws_ml[((bh * splits + s) * Sq + q) * 2]);
  float L = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (M != -INFINITY) {
    for (int s = 0; s < splits; ++s) {
      const long long slot = (bh * splits + s) * Sq + q;
      const float m = ws_ml[slot * 2];
      if (m == -INFINITY) continue;
      const float wgt = exp2f(m - M);
      L += ws_ml[slot * 2 + 1] * wgt;
      const float4 o = *reinterpret_cast<const float4*>(ws_o + slot * HD + v * 4);
      a0 += o.x * wgt; a1 += o.y * wgt; a2 += o.z * wgt; a3 += o.w * wgt;
    }
  }
  const float inv = L > 0.f ? 1.f / L : 0.f;
  const int b = static_cast<int>(bh / H), h = static_cast<int>(bh % H);
  bf16* dst = out + b * o_sb + h * o_sh + static_cast<long long>(q) * o_ss + v * 4;
  *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16(a0 * inv, a1 * inv), pack_bf16(a2 * inv, a3 * inv));
}

typedef CUresult (*PFN_encodeTiled2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled2 encode_fn() {
  static PFN_encodeTiled2 fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled2>(ptr);
  return fn;
}

// [B, S, H, D] view with element strides (sb, ss, sh), D contiguous -> 4-D map (d, s, h, b), box {64, rows, 1, 1}
static int make_qkv_map(CUtensorMap* m, const void* base, long long B, long long S, long long H, long long D,
                        long long sb, long long ss, long long sh, int box_rows) {
  PFN_encodeTiled2 fn = encode_fn();
  if (!fn) return VB_ERR_DRIVER;
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(D), static_cast<cuuint64_t>(S), static_cast<cuuint64_t>(H),
                        static_cast<cuuint64_t>(B)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(ss) * 2, static_cast<cuuint64_t>(sh) * 2, static_cast<cuuint64_t>(sb) * 2};
  cuuint32_t box[4] = {64, static_cast<cuuint32_t>(box_rows), 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? VB_OK : VB_ERR_DRIVER;
}

template <int HD, typename P>
static int launch_tc(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const P& p,
                     cudaStream_t stream) {
  constexpr int smem = tc_smem_bytes<HD>();
  static bool attr = false;
  auto kern = flash_attn_tc_kernel<HD, P>;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
    attr = true;
  }
  dim3 grid(((p.Sq + TC_BM - 1) / TC_BM) * p.splits, p.H, p.B);
  { cudaError_t le = vb_launch(kern, grid, dim3(TC_THREADS), smem, stream, tq, tk, tv, p); if (le != cudaSuccess) { vb_set_last_error(le); return VB_ERR_CUDA; } }
  if (p.splits > 1) {
    const long long items = static_cast<long long>(p.B) * p.H * p.Sq * (p.D / 4);
    cudaError_t le = vb_launch(attn_split_merge_kernel, dim3(static_cast<unsigned>((items + 255) / 256)), dim3(256), 0, stream,
                               static_cast<const float*>(p.ws_o), static_cast<const float*>(p.ws_ml), p.o, p.o_sb, p.o_ss, p.o_sh,
                               p.B, p.H, p.Sq, p.D, HD, p.splits);
    if (le != cudaSuccess) { vb_set_last_error(le); return VB_ERR_CUDA; }
  }
  VB_LAUNCH_CHECK();
  return VB_OK;
}

}  // namespace vb

using namespace vb;

// Diagnostics: {site id of the first timed-out wait (0 = none), packed block index, thread}; clears the record.
extern "C" int vb200_attention_watchdog(uint32_t* out3) {
  VB_CHECK_ARG(out3);
  unsigned int h[4] = {0, 0, 0, 0};
  cudaError_t e = cudaMemcpyFromSymbol(h, g_tc_watchdog, sizeof(h));
  if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
  out3[0] = h[0]; out3[1] = h[1]; out3[2] = h[2];
  if (h[0]) {
    unsigned int z[4] = {0, 0, 0, 0};
    cudaMemcpyToSymbol(g_tc_watchdog, z, sizeof(z));
  }
  return VB_OK;
}

// Resident CTAs per SM of the wgmma attention kernel (by registers / shared memory).
extern "C" int vb200_attention_tc_occupancy(int head_dim) {
  int n = 0;
  cudaError_t e;
  if (head_dim == 64) {
    constexpr int smem = tc_smem_bytes<64>();
    cudaFuncSetAttribute(flash_attn_tc_kernel<64, TcAttnParams>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, flash_attn_tc_kernel<64, TcAttnParams>, TC_THREADS, smem);
  } else if (head_dim == 128) {
    constexpr int smem = tc_smem_bytes<128>();
    cudaFuncSetAttribute(flash_attn_tc_kernel<128, TcAttnParams>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, flash_attn_tc_kernel<128, TcAttnParams>, TC_THREADS, smem);
  } else {
    return VB_ERR_ARG;
  }
  if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
  return n;
}

static int tc_hd(int64_t head_dim) { return head_dim <= 64 ? 64 : head_dim <= 128 ? 128 : 192; }

// split-KV factor: only when the (query tile, head, batch) grid leaves most SMs idle and there are enough key blocks
static int tc_splits(int64_t B, int64_t H, int64_t Sq, int64_t Skv, int causal) {
  if (causal) return 1;
  const long long ctas = ((Sq + TC_BM - 1) / TC_BM) * H * B;
  const long long nblk = (Skv + TC_BN - 1) / TC_BN;
  const int sms = vb_num_sms();
  if (ctas * 2 > sms || nblk < 8) return 1;
  long long s = (2LL * sms + ctas - 1) / ctas;
  if (s > nblk / 4) s = nblk / 4;
  if (s > 32) s = 32;
  return s < 2 ? 1 : static_cast<int>(s);
}

size_t vb_attention_tc_workspace(int64_t B, int64_t H, int64_t Sq, int64_t Skv, int64_t head_dim, int causal) {
  const int s = tc_splits(B, H, Sq, Skv, causal);
  if (s <= 1) return 0;
  return static_cast<size_t>(s) * B * H * Sq * (tc_hd(head_dim) + 2) * sizeof(float);
}

// Returns VB_ERR_UNSUPPORTED when the shape / strides are outside what this kernel handles; the caller
// (vb200_attention) then uses the mma.sync kernel.
int vb_attention_tc(const void* q, const void* k, const void* v, void* out, int64_t B, int64_t H, int64_t Sq,
                    int64_t Skv, int64_t head_dim, int64_t q_sb, int64_t q_ss, int64_t q_sh, int64_t k_sb,
                    int64_t k_ss, int64_t k_sh, int64_t v_sb, int64_t v_ss, int64_t v_sh, int64_t o_sb, int64_t o_ss,
                    int64_t o_sh, float scale, int causal, const int32_t* kv_len, const uint8_t* mask, int64_t m_sb,
                    int64_t m_sh, int64_t m_sq, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (head_dim != 40 && head_dim != 64 && head_dim != 80 && head_dim != 128 && head_dim != 160) return VB_ERR_UNSUPPORTED;
  if (Skv < 1 || Sq < 1) return VB_ERR_UNSUPPORTED;
  const int64_t st[12] = {q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh};
  for (int i = 0; i < 12; ++i)
    if (st[i] % 8 != 0 || st[i] < 0) return VB_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
       reinterpret_cast<uintptr_t>(out)) & 15)
    return VB_ERR_UNSUPPORTED;
  if (q_ss == 0 || k_ss == 0 || v_ss == 0) return VB_ERR_UNSUPPORTED;
  // a tensor-map dim of extent > 1 needs a non-zero stride: broadcast operands stay on the mma.sync kernel
  if ((B > 1 && (q_sb == 0 || k_sb == 0 || v_sb == 0)) || (H > 1 && (q_sh == 0 || k_sh == 0 || v_sh == 0)))
    return VB_ERR_UNSUPPORTED;
  // extent-1 dims still need a legal (16-byte multiple, non-zero) stride value
  auto fix = [](int64_t stride, int64_t fallback) { return stride == 0 ? fallback : stride; };
  CUtensorMap tq, tk, tv;
  if (int r = make_qkv_map(&tq, q, B, Sq, H, head_dim, fix(q_sb, q_ss * Sq), q_ss, fix(q_sh, q_ss * Sq), TC_BM)) return r;
  if (int r = make_qkv_map(&tk, k, B, Skv, H, head_dim, fix(k_sb, k_ss * Skv), k_ss, fix(k_sh, k_ss * Skv), TC_BN)) return r;
  if (int r = make_qkv_map(&tv, v, B, Skv, H, head_dim, fix(v_sb, v_ss * Skv), v_ss, fix(v_sh, v_ss * Skv), TC_BN)) return r;
  TcAttnParams p;
  p.o = reinterpret_cast<bf16*>(out);
  p.o_sb = o_sb; p.o_ss = o_ss; p.o_sh = o_sh;
  p.B = static_cast<int>(B); p.H = static_cast<int>(H); p.Sq = static_cast<int>(Sq); p.Skv = static_cast<int>(Skv);
  p.scale_log2 = scale * 1.4426950408889634f;
  p.causal = causal;
  p.kv_len = kv_len;
  p.D = static_cast<int>(head_dim);
  p.mask = mask;
  p.m_sb = m_sb; p.m_sh = m_sh; p.m_sq = m_sq;
  p.splits = 1;
  p.ws_o = nullptr;
  p.ws_ml = nullptr;
  const size_t need = vb_attention_tc_workspace(B, H, Sq, Skv, head_dim, causal);
  if (need > 0 && kv_len == nullptr && workspace != nullptr && workspace_bytes >= need && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0 &&
      (head_dim % 4) == 0) {
    p.splits = tc_splits(B, H, Sq, Skv, causal);
    p.ws_o = reinterpret_cast<float*>(workspace);
    p.ws_ml = p.ws_o + static_cast<size_t>(p.splits) * B * H * Sq * tc_hd(head_dim);
  }
  if (head_dim <= 64) return launch_tc<64>(tq, tk, tv, p, stream);
  if (head_dim <= 128) return launch_tc<128>(tq, tk, tv, p, stream);
  return launch_tc<192>(tq, tk, tv, p, stream);
}

// ---------------------------------------------------------------- paged prefill: a chunk of queries over the KV cache
// split-KV factor of the paged kernel: a chunk whose (query tile, head, batch) grid fills at most half the SMs (a one-user
// chat turn: 32 CTAs) has its key blocks divided so that the split grid still fits one wave of 2 CTAs per SM, at least
// 2 key blocks per split (a grid closer to one CTA per SM runs faster unsplit: the split one would need a second wave)
static int paged_splits(int64_t B, int64_t H, int64_t Sq, int64_t max_kv_len) {
  const long long ctas = ((Sq + TC_BM - 1) / TC_BM) * H * B;
  const long long nblk = (max_kv_len + TC_BN - 1) / TC_BN;
  const int sms = vb_num_sms();
  if (ctas * 2 > sms || nblk < 4) return 1;
  long long s = 2LL * sms / ctas;
  if (s > nblk / 2) s = nblk / 2;
  if (s > 32) s = 32;
  return s < 2 ? 1 : static_cast<int>(s);
}

extern "C" size_t vb200_attention_paged_workspace_size(int64_t B, int64_t H, int64_t Sq, int64_t head_dim,
                                                       int64_t max_kv_len) {
  if (B <= 0 || H <= 0 || Sq <= 0 || head_dim != 128 || max_kv_len <= 0) return 0;
  const int s = paged_splits(B, H, Sq, max_kv_len);
  if (s <= 1) return 0;
  return static_cast<size_t>(s) * B * H * Sq * (128 + 2) * sizeof(float);
}

extern "C" int vb200_attention_paged(const void* q, int64_t q_sb, int64_t q_ss, int64_t q_sh, const void* k_pages,
                                     const void* v_pages, int64_t num_pages, const int32_t* block_table, int64_t max_pages,
                                     const int32_t* q_start, const int32_t* q_len, void* out, int64_t o_sb, int64_t o_ss,
                                     int64_t o_sh, int64_t B, int64_t H, int64_t Sq, int64_t head_dim, int64_t page_size,
                                     int64_t max_kv_len, float scale, void* workspace, size_t workspace_bytes,
                                     cudaStream_t stream) {
  VB_CHECK_ARG(q && k_pages && v_pages && block_table && q_start && q_len && out);
  VB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && head_dim > 0 && page_size > 0 && num_pages > 0 && max_pages > 0);
  VB_CHECK_ARG(B <= 65535 && H <= 65535 && Sq <= (1LL << 30) && num_pages <= (1LL << 31) - 1 && max_pages <= (1LL << 24));
  VB_CHECK_ARG(max_kv_len > 0 && max_kv_len <= max_pages * page_size);
  const int64_t st[6] = {q_sb, q_ss, q_sh, o_sb, o_ss, o_sh};
  for (int i = 0; i < 6; ++i) VB_CHECK_ARG(st[i] >= 0 && st[i] % 8 == 0);
  VB_CHECK_ARG(q_ss > 0 && o_ss > 0);
  VB_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(k_pages) |
                 reinterpret_cast<uintptr_t>(v_pages)) & 15) == 0);
  if (head_dim != 128 || page_size != TC_BN) return VB_ERR_UNSUPPORTED;
  // a tensor-map dim of extent > 1 needs a non-zero stride (as in vb_attention_tc)
  VB_CHECK_ARG((B == 1 || q_sb > 0) && (H == 1 || q_sh > 0));
  auto fix = [](int64_t stride, int64_t fallback) { return stride == 0 ? fallback : stride; };
  const int64_t page_elems = TC_BN * head_dim;
  CUtensorMap tq, tk, tv;
  if (int r = make_qkv_map(&tq, q, B, Sq, H, head_dim, fix(q_sb, q_ss * Sq), q_ss, fix(q_sh, q_ss * Sq), TC_BM)) return r;
  // the cache as [num_pages, 64 keys, H, D] views: coordinate (d, key, head, page)
  if (int r = make_qkv_map(&tk, k_pages, num_pages, TC_BN, H, head_dim, H * page_elems, head_dim, page_elems, TC_BN)) return r;
  if (int r = make_qkv_map(&tv, v_pages, num_pages, TC_BN, H, head_dim, H * page_elems, head_dim, page_elems, TC_BN)) return r;
  TcPagedParams p;
  p.o = reinterpret_cast<bf16*>(out);
  p.o_sb = o_sb; p.o_ss = o_ss; p.o_sh = o_sh;
  p.B = static_cast<int>(B); p.H = static_cast<int>(H); p.Sq = static_cast<int>(Sq);
  p.Skv = static_cast<int>(max_kv_len);
  p.D = static_cast<int>(head_dim);
  p.scale_log2 = scale * 1.4426950408889634f;
  p.causal = 1;
  p.kv_len = nullptr;
  p.mask = nullptr;
  p.m_sb = p.m_sh = p.m_sq = 0;
  p.block_table = block_table;
  p.max_pages = static_cast<int>(max_pages);
  p.q_start = q_start;
  p.q_len = q_len;
  p.max_kv_len = static_cast<int>(max_kv_len);
  p.splits = 1;
  p.ws_o = nullptr;
  p.ws_ml = nullptr;
  const size_t need = vb200_attention_paged_workspace_size(B, H, Sq, head_dim, max_kv_len);
  if (need > 0 && workspace != nullptr && workspace_bytes >= need && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0) {
    p.splits = paged_splits(B, H, Sq, max_kv_len);
    p.ws_o = reinterpret_cast<float*>(workspace);
    p.ws_ml = p.ws_o + static_cast<size_t>(p.splits) * B * H * Sq * 128;
  }
  return launch_tc<128>(tq, tk, tv, p, stream);
}
