// vitron_b200 — bf16 GEMM / implicit-GEMM convolution on sm_90a warpgroup MMA (wgmma) fed by TMA through mbarriers.
//
//   D[M, N] = epilogue( A[M, K] · B[N, K]^T )        (both operands K-major, fp32 accumulate)
//
// One persistent kernel of three warpgroups:
//   warpgroup 0      TMA producer (one thread): A / B k-blocks into a ring of 128B-swizzled shared-memory stages
//   warpgroups 1, 2  consumers: tile rows [64 (wg - 1), +64) — wgmma m64 n BLOCK_N k16 straight from the ring, the
//                    accumulators in registers, then the fused epilogue from registers to global memory
// setmaxnreg hands the producer's registers to the consumers (a 128 x 256 tile is 128 fp32 accumulators per thread).
// Each consumer keeps one k-block of MMAs in flight and releases a ring slot as soon as the MMAs reading it retire, so the
// producer runs ahead into the next tile while the consumers are in their epilogue. wgmma.wait_group only covers the
// executing warp's share of the MMA, so every consumer warp arrives on the slot's empty barrier (8 arrivals per slot).
//
// The A operand comes either from a plain 2-D row-major matrix or, for convolutions, straight from the NHWC activation
// through a 4-D tensor map: every (tap, channel-chunk) k-step is one TMA box {64 ch, TW, TH, TN} fetched at the
// tap-shifted coordinate, out-of-bounds pixels are zero-filled by the TMA unit (= zero padding), so no im2col buffer
// exists. A box of fewer than 128 pixels leaves stale rows in the stage: they only feed accumulator rows that are never
// stored (tile_row_to_orow).
//
// Epilogue features are TEMPLATE flags (F_*): a variant only contains the code of the features it was instantiated with;
// F_ALL / F_ALL_GLU resolve every feature at run time (the generic variants, vb200_set_gemm_impl(1)).
// RESB ("resident B"): for small K the CTA keeps ALL k-blocks of ONE n-block of the weight matrix in shared memory and
// walks m-tiles of that n-block only; the ring then carries A alone. Without it every 128 x BN tile re-fetches its B tile
// from L2, which bounds the small-K UNet GEMMs (K = 320: 40 KB of B per 16 KB A k-block at BN = 160).
// Split-K (F_WS) and swap-AB write raw fp32 partials to the workspace, indexed by OUTPUT row (convolutions: output
// pixel); splitk_reduce_kernel (gemm.cu) sums them in split order and applies the epilogue.
//
// Covers (reference file:line in DESIGN.md): LLaMA q/k/v/o/gate/up/down/lm_head, CLIP ViT q/k/v/out/fc1/fc2,
// mm_projector, region MLP, every Linear / Conv2d(3x3,1x1) / Conv3d(3,1,1) of UNetSD_I2VGen, SEEM FPN convs + mask
// einsum, GLIGEN fuser linears.
#pragma once
#include "gemm_common.cuh"
#include "wgmma.cuh"

namespace vb {

// epilogue feature flags of a variant
constexpr int F_RS = 1;    // per-row fp32 scale (folded RMSNorm)
constexpr int F_RB = 2;    // per-row-group bias (time embedding of a ResBlock conv)
constexpr int F_RES = 4;   // out = residual + alpha * v   (residual may be null: out = alpha * v)
constexpr int F_ACT = 8;   // activation selected at run time (p.act)
constexpr int F_GLU = 16;  // packed SwiGLU / GEGLU selected at run time (p.glu)
constexpr int F_F32 = 32;  // fp32 output
constexpr int F_WS = 64;   // raw fp32 partials -> workspace (split-K, swap-AB), reduced by splitk_reduce_kernel
constexpr int F_ALL = F_RS | F_RB | F_RES | F_ACT | F_F32;            // every non-GLU feature at run time
constexpr int F_ALL_GLU = F_GLU | F_RS | F_RB | F_RES | F_F32;        // every GLU combination at run time

template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// output row (C orientation) of accumulator row r of m-block m_blk; -1 = padding row of the tile
__device__ __forceinline__ int tile_row_to_orow(const GemmParams& p, int m_blk, int r) {
  if (p.a_mode == 0) {
    const int g = m_blk * BLOCK_M + r;
    return g < p.M ? g : -1;
  }
  const int tiw = m_blk % p.tiles_w;
  const int rest = m_blk / p.tiles_w;
  const int tih = rest % p.tiles_h;
  const int tin = rest / p.tiles_h;
  const int tx = r % p.tw;
  const int r2 = r / p.tw;
  const int ty = r2 % p.th;
  const int tz = r2 / p.th;
  const int x = tiw * p.tw + tx, y = tih * p.th + ty, n = tin * p.tn + tz;
  if (tz < p.tn && x < p.wo && y < p.ho && n < p.nb) return (n * p.ho + y) * p.wo + x;
  return -1;
}

// two adjacent outputs (columns oc, oc + 1; the second only when `two`) of one row: residual / alpha, then the store
template <int F>
__device__ __forceinline__ void epi_store2(const GemmParams& p, int orow, int oc, bool two, bool vec, float v0, float v1) {
  if constexpr ((F & F_RES) != 0) {
    if (p.residual != nullptr) {
      // the residual may alias the output (in-place "z += f(z)"): plain coherent loads
      const bf16* rp = p.residual + static_cast<size_t>(orow) * p.ldr + oc;
      v0 = fmaf(p.alpha, v0, __bfloat162float(rp[0]));
      if (two) v1 = fmaf(p.alpha, v1, __bfloat162float(rp[1]));
    } else {
      v0 *= p.alpha;
      v1 *= p.alpha;
    }
  }
  if ((F & F_F32) != 0 && p.out_fp32) {
    float* dst = reinterpret_cast<float*>(p.out) + static_cast<size_t>(orow) * p.ldo + oc;
    if (two && vec) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
    else { dst[0] = v0; if (two) dst[1] = v1; }
  } else {
    bf16* dst = reinterpret_cast<bf16*>(p.out) + static_cast<size_t>(orow) * p.ldo + oc;
    if (two && vec) *reinterpret_cast<uint32_t*>(dst) = pack_bf16(v0, v1);
    else { dst[0] = __float2bfloat16(v0); if (two) dst[1] = __float2bfloat16(v1); }
  }
}

template <int BLOCK_N, int STAGES, int F, bool RESB = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_v2_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmParams p) {
  constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  constexpr int STAGE_BYTES = RESB ? A_BYTES : A_BYTES + B_BYTES;
  constexpr bool WS = (F & F_WS) != 0;
  constexpr bool GLU = (F & F_GLU) != 0;
  constexpr int NACC = BLOCK_N / 2;       // accumulators per consumer thread (64 x BLOCK_N over 128 threads)
  static_assert(BLOCK_N % 32 == 0, "tiles are whole 32-column GLU blocks");
  static_assert(B_BYTES % 1024 == 0, "stages stay 1024-byte aligned (128B swizzle atoms)");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem_al = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                                ~static_cast<uintptr_t>(1023));
  uint8_t* sB_res = smem_al;                                                    // RESB: [num_k_blocks][BLOCK_N x 128 B]
  uint8_t* smem = smem_al + (RESB ? p.num_k_blocks * B_BYTES : 0);              // the ring
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* b_full = empty_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;

  // Programmatic dependent launch: barrier set-up touches no global data; every global read and write follows pdl_wait().
  pdl_trigger();
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // one arrival per consumer warp (wgmma.wait_group completes per warp)
    }
    mbar_init(b_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  // work units of this CTA: (m-block, n-block, split) in grouped raster order, or — RESB — the m-blocks
  // m = blockIdx.x / n_blocks, += gridDim.x / n_blocks of the ONE n-block blockIdx.x % n_blocks (grid is a multiple of n_blocks)
  const int total_units = RESB ? p.m_blocks : p.m_blocks * p.n_blocks * p.splits;
  const int unit_first = RESB ? static_cast<int>(blockIdx.x) / p.n_blocks : static_cast<int>(blockIdx.x);
  const int unit_step = RESB ? static_cast<int>(gridDim.x) / p.n_blocks : static_cast<int>(gridDim.x);
  const int my_n_blk = RESB ? static_cast<int>(blockIdx.x) % p.n_blocks : 0;
  auto work_of = [&](int unit) {
    if constexpr (RESB) {
      TileCoord t;
      t.m_blk = unit; t.n_blk = my_n_blk; t.split = 0;
      return t;
    } else {
      return decode_work(p, unit);
    }
  };

  if (wg == 0) {
    // ===================================================== TMA producer
    setmaxnreg_dec<40>();
    if (tid == 0) {
      int stage = 0;
      uint32_t phase = 0;
      if constexpr (RESB) {
        mbar_arrive_expect_tx(b_full, static_cast<uint32_t>(p.num_k_blocks) * B_BYTES);
        for (int kb = 0; kb < p.num_k_blocks; ++kb)
          tma_load_2d(sB_res + kb * B_BYTES, &tmap_b, b_full, kb * BLOCK_K, my_n_blk * BLOCK_N);
      }
      for (int unit = unit_first; unit < total_units; unit += unit_step) {
        const TileCoord t = work_of(unit);
        int k0, k1;
        split_range(p, t.split, k0, k1);
        int cw = 0, ch = 0, cn = 0;
        if (p.a_mode == 1) {
          const int tiw = t.m_blk % p.tiles_w;
          const int rest = t.m_blk / p.tiles_w;
          cw = tiw * p.tw * p.stride - p.pad_w;
          ch = (rest % p.tiles_h) * p.th * p.stride - p.pad_h;
          cn = (rest / p.tiles_h) * p.tn;
        }
        for (int kb = k0; kb < k1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], p.a_box_bytes + (RESB ? 0 : B_BYTES));
          if (p.a_mode == 0) {
            tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BLOCK_K, t.m_blk * BLOCK_M);
          } else {
            const int tap = kb / p.cin_chunks;
            const int cc = kb - tap * p.cin_chunks;
            const int dy = tap / p.kw, dx = tap - dy * p.kw;
            tma_load_4d(sa, &tmap_a, &full_bar[stage], cc * BLOCK_K, cw + dx, ch + dy, cn);
          }
          if constexpr (!RESB) tma_load_2d(sa + A_BYTES, &tmap_b, &full_bar[stage], kb * BLOCK_K, t.n_blk * BLOCK_N);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================================================== consumers: MMA + epilogue
  setmaxnreg_inc<232>();
  const int cwg = wg - 1;                 // rows [64 cwg, +64) of every tile
  const int lane = tid & 31;
  float acc[NACC];
  int stage = 0;
  uint32_t phase = 0;
  if constexpr (RESB) {
    if (unit_first < total_units) mbar_wait(b_full, 0);
  }
  // accumulator fragment: acc[4i + 2h + e] = tile row r_lo + 8h, column 8i + cq + e
  const int r_lo = cwg * 64 + (tid >> 5) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const int esz = ((F & F_F32) != 0 && p.out_fp32) ? 4 : 2;
  const bool ovec = !WS && ((reinterpret_cast<uintptr_t>(p.out) | static_cast<uintptr_t>(p.ldo * esz)) & (2 * esz - 1)) == 0;
  const bool wvec = WS && !p.swap && ((reinterpret_cast<uintptr_t>(p.ws) | static_cast<uintptr_t>(p.ws_ld * 4)) & 7) == 0;

  for (int unit = unit_first; unit < total_units; unit += unit_step) {
    const TileCoord t = work_of(unit);
    int k0, k1;
    split_range(p, t.split, k0, k1);
    if (k1 <= k0) {
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    }
    int held = -1;   // ring slot whose MMAs may still be in flight
    for (int kb = k0; kb < k1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + cwg * (64 * 128);
      const uint32_t sb = RESB ? smem_u32(sB_res + kb * B_BYTES) : smem_u32(smem + stage * STAGE_BYTES + A_BYTES);
      const uint64_t da = gmma_desc_kmajor(sa), db = gmma_desc_kmajor(sb);
      wgmma_fence_operand(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
        Wgmma<BLOCK_N>::ss(acc, da + 2 * k, db + 2 * k, (kb > k0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_fence_operand(acc);
      wgmma_wait<1>();   // the previous k-block's MMAs have retired: its slot can be refilled
      if (held >= 0 && lane == 0) mbar_arrive(&empty_bar[held]);
      held = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_operand(acc);
    if (held >= 0 && lane == 0) mbar_arrive(&empty_bar[held]);

    // ---------------- epilogue, straight from the accumulator registers
    if (p.dbg & 1) continue;
    const int col0 = t.n_blk * BLOCK_N;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int orow = tile_row_to_orow(p, t.m_blk, r_lo + 8 * h);
      if (orow < 0) continue;
      if constexpr (WS) {
        float* wsp = p.ws + static_cast<size_t>(t.split) * p.ws_split_stride;
#pragma unroll
        for (int i = 0; i < BLOCK_N / 8; ++i) {
          const int col = col0 + 8 * i + cq;
          const float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
          if (col >= p.N) continue;
          const bool two = col + 1 < p.N;
          if (p.swap) {
            // C[token = col, feature = orow]
            wsp[static_cast<size_t>(col) * p.ws_ld + orow] = v0;
            if (two) wsp[static_cast<size_t>(col + 1) * p.ws_ld + orow] = v1;
          } else {
            float* dst = wsp + static_cast<size_t>(orow) * p.ws_ld + col;
            if (two && wvec) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
            else { dst[0] = v0; if (two) dst[1] = v1; }
          }
        }
      } else {
        float rs = 1.f;
        if constexpr ((F & F_RS) != 0) {
          if (p.rowscale != nullptr) rs = __ldg(p.rowscale + orow);
        }
        const bf16* rb = nullptr;
        if constexpr ((F & F_RB) != 0) {
          if (p.rowbias != nullptr) rb = p.rowbias + static_cast<size_t>(orow / p.rowbias_rows) * p.N;
        }
        auto add_bias = [&](int col, float v) {
          if (p.bias != nullptr) v += __bfloat162float(p.bias[col]);
          if constexpr ((F & F_RB) != 0) {
            if (rb != nullptr) v += __bfloat162float(rb[col]);
          }
          return v;
        };
        if constexpr (GLU) {
          // packed GLU: accumulator columns come in blocks of 32 = [16 x "a" | 16 x "b"] (N % 32 == 0); the "a" and "b"
          // values of an output sit in the same thread, 8 fragment columns apart
#pragma unroll
          for (int q = 0; q < BLOCK_N / 32; ++q) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              const int ia = 4 * (4 * q + j) + 2 * h, ib = ia + 8;
              const int ca = col0 + 32 * q + 8 * j + cq;
              if (ca >= p.N) continue;
              const float a0 = add_bias(ca, acc[ia] * rs), a1 = add_bias(ca + 1, acc[ia + 1] * rs);
              const float b0 = add_bias(ca + 16, acc[ib] * rs), b1 = add_bias(ca + 17, acc[ib + 1] * rs);
              float o0, o1;
              if (p.glu == VB_GLU_SWIGLU) { o0 = silu(a0) * b0; o1 = silu(a1) * b1; }
              else { o0 = a0 * gelu_erf_fast(b0); o1 = a1 * gelu_erf_fast(b1); }
              epi_store2<F>(p, orow, (col0 + 32 * q) / 2 + 8 * j + cq, true, ovec, o0, o1);
            }
          }
        } else {
#pragma unroll
          for (int i = 0; i < BLOCK_N / 8; ++i) {
            const int col = col0 + 8 * i + cq;
            if (col >= p.N) continue;
            const bool two = col + 1 < p.N;
            float v0 = add_bias(col, acc[4 * i + 2 * h] * rs);
            float v1 = two ? add_bias(col + 1, acc[4 * i + 2 * h + 1] * rs) : 0.f;
            if constexpr ((F & F_ACT) != 0) {
              v0 = apply_act(v0, p.act);
              v1 = apply_act(v1, p.act);
            }
            epi_store2<F>(p, orow, col, two, ovec, v0, v1);
          }
        }
      }
    }
  }
}

// shared memory of a launch: [RESB: B slab] + ring + barriers (+ 1 KB for the manual 1024-byte alignment)
template <int BN, int STAGES, bool RESB>
constexpr int gemm_smem(int nkb) {
  return (RESB ? nkb * BN * BLOCK_K * 2 : 0) + STAGES * (BLOCK_M * BLOCK_K * 2 + (RESB ? 0 : BN * BLOCK_K * 2)) + 1024 + 256;
}

template <int BN, int STAGES, int F>
int launch_v2_resb(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  const int smem = gemm_smem<BN, STAGES, true>(p.num_k_blocks);
  if (smem > SMEM_LIMIT || p.a_mode != 0 || p.splits != 1) return VB_ERR_UNSUPPORTED;
  static bool attr_set = false;
  auto kern = gemm_v2_kernel<BN, STAGES, F, true>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
    attr_set = true;
  }
  // whole CTA groups of n_blocks: every CTA owns one n-block, its m-blocks are strided over the groups
  int groups = vb_num_sms() / p.n_blocks;
  if (groups < 1) return VB_ERR_UNSUPPORTED;
  if (groups > p.m_blocks) groups = p.m_blocks;
  const int grid = groups * p.n_blocks;
  cudaError_t le = vb_launch(kern, dim3(grid), dim3(GEMM_THREADS), smem, stream, ta, tb, p);
  if (le != cudaSuccess) { vb_set_last_error(le); return VB_ERR_CUDA; }
  return VB_OK;
}

template <int BN, int STAGES, int F>
int launch_v2(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  constexpr int smem = gemm_smem<BN, STAGES, false>(0);
  static_assert(smem <= SMEM_LIMIT, "smem budget");
  static bool attr_set = false;
  auto kern = gemm_v2_kernel<BN, STAGES, F>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
    attr_set = true;
  }
  const int units = p.m_blocks * p.n_blocks * p.splits;
  const int grid = units < vb_num_sms() ? units : vb_num_sms();
  cudaError_t le = vb_launch(kern, dim3(grid), dim3(GEMM_THREADS), smem, stream, ta, tb, p);
  if (le != cudaSuccess) { vb_set_last_error(le); return VB_ERR_CUDA; }
  return VB_OK;
}

// resident-B variants exist for the feature sets of the small-K UNet / ViT GEMMs; RSTAGES = A-ring depth next to the B slab
template <int BN, int RSTAGES>
int dispatch_v2_resb(int need, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  if (need == 0) return launch_v2_resb<BN, RSTAGES, 0>(ta, tb, p, stream);
  if (need == F_RES) return launch_v2_resb<BN, RSTAGES, F_RES>(ta, tb, p, stream);
  if (need == F_GLU) return launch_v2_resb<BN, RSTAGES, F_GLU>(ta, tb, p, stream);
  if (need == F_ACT) return launch_v2_resb<BN, RSTAGES, F_ACT>(ta, tb, p, stream);
  return VB_ERR_UNSUPPORTED;
}

// variant of tile width BN covering the feature set `need` (F_* mask; F_WS selects the partials variant); `generic`
// takes the variants that resolve every feature at run time
template <int BN, int STAGES>
int dispatch_v2(int need, bool generic, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  if (need & F_WS) return launch_v2<BN, STAGES, F_WS>(ta, tb, p, stream);
  if (!generic) {
    if (need == 0) return launch_v2<BN, STAGES, 0>(ta, tb, p, stream);
    if (need == F_ACT) return launch_v2<BN, STAGES, F_ACT>(ta, tb, p, stream);
    if (need == F_RES) return launch_v2<BN, STAGES, F_RES>(ta, tb, p, stream);
    if (need == F_GLU) return launch_v2<BN, STAGES, F_GLU>(ta, tb, p, stream);
    if (need == (F_GLU | F_RS)) return launch_v2<BN, STAGES, F_GLU | F_RS>(ta, tb, p, stream);
    if (need == F_RS) return launch_v2<BN, STAGES, F_RS>(ta, tb, p, stream);
    if (need == F_RB) return launch_v2<BN, STAGES, F_RB>(ta, tb, p, stream);
  }
  if (need & F_GLU) return launch_v2<BN, STAGES, F_ALL_GLU>(ta, tb, p, stream);
  return launch_v2<BN, STAGES, F_ALL>(ta, tb, p, stream);
}

int launch_gemm_v2_resb(int bn, int need, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream);
int launch_gemm_v2_256(int need, bool generic, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream);
int launch_gemm_v2_160(int need, bool generic, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream);
int launch_gemm_v2_128(int need, bool generic, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream);
int launch_gemm_v2_64(int need, bool generic, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream);
int launch_gemm_v2_32(int need, bool generic, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream);

}  // namespace vb
