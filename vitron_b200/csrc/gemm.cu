// vitron_b200 — host side of the bf16 GEMM / implicit-GEMM convolution (kernel: gemm_v2.cuh, wgmma + TMA, sm_90a):
// tile-width / split-K planning, tensor maps, the split-K / swap-AB reduce kernel and the C ABI entry points.
#include <cstdlib>
#include "gemm_v2.cuh"

namespace vb {

// ------------------------------------------------------------------ split-K / swap reduce
// out[m, n'] = epilogue( sum_s ws[s, m, n] ), same epilogue semantics as the fused path.
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, int splits,
                                     long long split_stride, long long ws_ld, int rows, int ncols,
                                     void* out, long long ldo, const bf16* __restrict__ bias,
                                     const bf16* __restrict__ rowbias, int rowbias_rows,
                                     const bf16* __restrict__ residual, long long ldr, float alpha,
                                     int act, int glu, int out_fp32, const float* __restrict__ rowscale) {
  pdl_trigger();
  pdl_wait();
  const int n_out_total = glu != VB_GLU_NONE ? ncols / 2 : ncols;
  const int groups = (n_out_total + 7) / 8;
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(rows) * groups) return;
  reduce_item(ws, splits, split_stride, ws_ld, static_cast<int>(idx / groups), static_cast<int>(idx % groups) * 8,
              ncols, out, ldo, bias, rowbias, rowbias_rows, residual, ldr, alpha, act, glu, out_fp32, rowscale);
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(p);
  return fn;
}

static int make_tmap(CUtensorMap* m, const void* ptr, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box,
                     const uint32_t* estr, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return VB_ERR_DRIVER;
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), dims,
                  strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? VB_OK : VB_ERR_DRIVER;
}


static int swap_splits(long long M, long long N, long long K) {
  // maximise (CTA wave utilisation) x (k-block balance across splits); fewer splits win ties
  const int sms = vb_num_sms();
  const int m_blocks = static_cast<int>((N + BLOCK_M - 1) / BLOCK_M);
  const int kblocks = static_cast<int>((K + BLOCK_K - 1) / BLOCK_K);
  int best = 1;
  float best_score = -1.f;
  for (int s = 1; s <= 32 && s <= kblocks; ++s) {
    if (static_cast<size_t>(s) * M * N * sizeof(float) > (static_cast<size_t>(96) << 20)) break;
    const long long units = static_cast<long long>(m_blocks) * s;
    const long long waves = (units + sms - 1) / sms;
    const float util = static_cast<float>(units) / static_cast<float>(waves * sms);
    const int per = (kblocks + s - 1) / s;
    const float bal = static_cast<float>(kblocks) / static_cast<float>(s * per);
    // every extra wave / split costs a fixed ramp (pipeline fill, partial write + reduction)
    const float score = util * bal - 0.01f * static_cast<float>(s);
    if (score > best_score + 1e-6f) { best_score = score; best = s; }
  }
  return best;
}

static int validate_epi(const vb_epilogue* e, long long N) {
  if (e->glu != VB_GLU_NONE && (N % 32) != 0) return VB_ERR_ARG;
  if (e->act < VB_ACT_NONE || e->act > VB_ACT_SILU) return VB_ERR_ARG;
  if (e->glu < VB_GLU_NONE || e->glu > VB_GLU_GEGLU) return VB_ERR_ARG;
  return VB_OK;
}

// ------------------------------------------------------------------ planning
static int g_gemm_impl = 0;  // 0: epilogue variants specialised by feature set, 1: the run-time-feature variants only
static int g_gemm_resb = 1;  // resident-B variant: bit 0 = K <= 320 (5 k-blocks), bit 1 = also K <= 640 at BN = 128; 0 = off
static int g_gemm_dbg = 0;   // GemmParams.dbg (measurement aid)
int resb_smem_bytes(int bn, int nkb);  // gemm_v2_resb.cu

// Tile width of the resident-B variant for M x N x (nkb k-blocks), or 0 when it does not apply: the widest slab that
// fits next to an A ring deep enough to cover the L2 latency (BN = 160 with 6 A stages at K <= 320; BN = 128 at K <= 640).
static int resb_tile(long long M, long long N, int nkb, int need) {
  if (g_gemm_impl == 1 || !(g_gemm_resb & 3) || (need != 0 && need != F_RES && need != F_GLU && need != F_ACT)) return 0;
  if (nkb > 5 && !(g_gemm_resb & 2)) return 0;
  if (M < 4096) return 0;                       // few m-tiles: nothing to amortise the slab load over
  const int cands[3] = {160, 256, 128};
  int best = 0;
  float best_cost = 1e30f;
  for (int i = 0; i < 3; ++i) {
    const int bn = cands[i];
    if (resb_smem_bytes(bn, nkb) > SMEM_LIMIT) continue;
    const long long nb = (N + bn - 1) / bn;
    if (nb > vb_num_sms()) continue;
    const int groups = vb_num_sms() / static_cast<int>(nb);
    const long long mb = (M + BLOCK_M - 1) / BLOCK_M;
    const long long per_cta = (mb + groups - 1) / groups;     // m-tiles of the busiest CTA
    // per tile and k-block: MMA ~ bn / 256, A stream ~ 0.55 with a deep A ring (BN 160), 0.9 with 3 stages (model weights)
    const float mma = static_cast<float>(bn) / 256.f, astream = bn == 160 ? 0.55f : 0.9f;
    const float cost = static_cast<float>(per_cta) * nkb * (mma > astream ? mma : astream);
    if (cost < best_cost) { best_cost = cost; best = bn; }
  }
  return best;
}

struct TilePlan {
  int bn, splits;
};

// Tile width and split-K factor for `mb` 128-row m-blocks x N columns x `kblocks` k-steps. Time model in units of one
// 128x256x64 k-step: per-unit main loop = k-steps x tk[bn] (narrow tiles re-read A from shared memory more often per
// MMA and carry the fixed per-k-step cost of the pipeline), waves = ceil(units / SMs); a split costs its partial write +
// the reduce kernel. The weights here, in resb_tile and in swap_splits are NOT calibrated on H100: they are the relative
// costs of the earlier tcgen05 kernel, kept as a starting point; tools/bn_sweep.py measures the per-width times to re-fit them.
static TilePlan plan_tiles(long long mb, long long N, int kblocks, bool allow_split, long long out_rows) {
  const int sms = vb_num_sms();
  const int cands[5] = {256, 160, 128, 64, 32};
  const float tk[5] = {1.0f, 0.78f, 0.76f, 0.625f, 0.57f};
  TilePlan best = {256, 1};
  float best_t = 1e30f;
  if (const char* force = getenv("VB200_FORCE_BN")) {  // tuning knob for tools/bn_sweep.py
    const int v = atoi(force);
    if (v == 256 || v == 160 || v == 128 || v == 64 || v == 32) return {v, 1};
  }
  for (int i = 0; i < 5; ++i) {
    const int bn = cands[i];
    const long long nbk = (N + bn - 1) / bn;
    const long long tiles = mb * nbk;
    for (int sp = 1; sp <= 8; ++sp) {
      if (sp > 1) {
        if (!allow_split || tiles * 10 >= static_cast<long long>(sms) * 7) break;
        if (kblocks / sp < 4) break;
        if (static_cast<unsigned long long>(sp) * out_rows * N * sizeof(float) > (64ull << 20)) break;
      }
      const long long units = tiles * sp;
      const long long waves = (units + sms - 1) / sms;
      const int kpu = (kblocks + sp - 1) / sp;
      float t = static_cast<float>(waves) * (kpu * tk[i] + (sp > 1 ? 1.5f : 0.f));
      t += 2.0f * bn / 256.f;
      // a split writes and re-reads sp fp32 copies of the output through L2 and pays one more launch
      if (sp > 1) t += static_cast<float>(sp) * out_rows * N * 8.0f / 5.0e6f / 0.27f + 9.0f;
      if (t < best_t - 1e-4f) { best_t = t; best = {bn, sp}; }
    }
  }
  return best;
}

static int v2_need(const vb_epilogue* e, int splits) {
  if (splits > 1) return F_WS;
  int need = 0;
  if (e->rowscale) need |= F_RS;
  if (e->rowbias) need |= F_RB;
  if (e->residual || e->alpha != 1.0f) need |= F_RES;
  if (e->act != VB_ACT_NONE) need |= F_ACT;
  if (e->glu != VB_GLU_NONE) need |= F_GLU;
  if (e->out_fp32) need |= F_F32;
  return need;
}

static int launch_gemm_v2(int bn, int need, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                          cudaStream_t stream) {
  const bool generic = g_gemm_impl == 1;
  int r;
  switch (bn) {
    case 256: r = launch_gemm_v2_256(need, generic, ta, tb, p, stream); break;
    case 160: r = launch_gemm_v2_160(need, generic, ta, tb, p, stream); break;
    case 128: r = launch_gemm_v2_128(need, generic, ta, tb, p, stream); break;
    case 64: r = launch_gemm_v2_64(need, generic, ta, tb, p, stream); break;
    case 32: r = launch_gemm_v2_32(need, generic, ta, tb, p, stream); break;
    default: return VB_ERR_ARG;
  }
  if (r != VB_OK || !(need & F_WS)) return r;
  // split-K / swap-AB: sum the partials in split order + the fused epilogue, one thread per 8 outputs of a row
  // (C orientation: swap-AB partials are [token, feature] like the plain ones)
  const int rows = p.swap ? p.N : p.M, cols = p.swap ? p.M : p.N;
  const int n_out = p.glu != VB_GLU_NONE ? cols / 2 : cols;
  const long long items = static_cast<long long>(rows) * ((n_out + 7) / 8);
  cudaError_t le = vb_launch(splitk_reduce_kernel, dim3(static_cast<unsigned>((items + 255) / 256)), dim3(256), 0, stream,
                             static_cast<const float*>(p.ws), p.splits, p.ws_split_stride, p.ws_ld, rows, cols, p.out, p.ldo, p.bias,
                             p.rowbias, p.rowbias_rows, p.residual, p.ldr, p.alpha, p.act, p.glu, p.out_fp32, p.rowscale);
  if (le != cudaSuccess) { vb_set_last_error(le); return VB_ERR_CUDA; }
  return VB_OK;
}

// conv output-pixel tile tw x th x tn (<= 128 accumulator rows): the shape that covers the output with the fewest
// tiles; ties go to the widest tile (longest contiguous runs for the TMA boxes)
static void conv_pixel_tile(int wo, int ho, long long nb, int& tw, int& th, int& tn) {
  tw = th = tn = 1;
  long long best = -1;
  for (int cw = wo < 128 ? wo : 128; cw >= 1; --cw) {
    const int hmax = 128 / cw < ho ? 128 / cw : ho;
    for (int ch = hmax; ch >= 1; --ch) {
      int cn = 128 / (cw * ch);
      if (cn > nb) cn = static_cast<int>(nb);
      const long long blocks = static_cast<long long>((wo + cw - 1) / cw) * ((ho + ch - 1) / ch) * ((nb + cn - 1) / cn);
      if (best < 0 || blocks < best) { best = blocks; tw = cw; th = ch; tn = cn; }
    }
  }
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static void set_epilogue(GemmParams& p, const vb_epilogue* epi) {
  p.bias = reinterpret_cast<const bf16*>(epi->bias);
  p.rowbias = reinterpret_cast<const bf16*>(epi->rowbias);
  p.rowbias_rows = epi->rowbias_rows > 0 ? static_cast<int>(epi->rowbias_rows) : 1;
  p.residual = reinterpret_cast<const bf16*>(epi->residual);
  p.ldr = epi->ldr;
  p.alpha = epi->alpha;
  p.act = epi->act;
  p.glu = epi->glu;
  p.out_fp32 = epi->out_fp32;
  p.rowscale = epi->rowscale;
  p.dbg = g_gemm_dbg;
}

}  // namespace vb

using namespace vb;

extern "C" int vb200_set_gemm_debug(int resident_b, int dbg) {
  const int prev = g_gemm_resb | (g_gemm_dbg << 8);
  if (resident_b >= 0) g_gemm_resb = resident_b;
  if (dbg >= 0) g_gemm_dbg = dbg;
  return prev;
}

extern "C" int vb200_set_gemm_impl(int impl) {
  const int prev = g_gemm_impl;
  if (impl == 0 || impl == 1) g_gemm_impl = impl;
  return prev;
}

int vb_launch_gemv(const void* A, int64_t lda, const void* W, int64_t ldw, void* out, int64_t ldo, int64_t M,
                   int64_t N, int64_t K, const vb_epilogue* e, cudaStream_t stream);  // gemv.cu

// 17..64 rows: swap-AB + split-K (weights in the 128-row tile slot, every SM streams a K slice) pays off only when the
// weight matrix is large enough to be an HBM stream (LLM decode at batch 17..64: 33-180 MB per GEMM); the small matrices of
// the SEEM / GLIGEN token paths run on the persistent kernel with a mostly empty 128-row tile (one launch instead of two).
static bool use_swap(int64_t M, int64_t N, int64_t K) { return M <= 64 && N * K > (4ll << 20); }

extern "C" size_t vb200_gemm_bf16_workspace_size(int64_t M, int64_t N, int64_t K) {
  // M <= 16: weight-streaming kernel (gemv.cu), no workspace; 16 < M <= 64 and a long weight stream: swap-AB + split-K
  if (M <= 16 || N <= 0 || K <= 0) return 0;
  if (use_swap(M, N, K))
    return static_cast<size_t>(swap_splits(M, N, K)) * static_cast<size_t>(M) * static_cast<size_t>(N) * sizeof(float);
  // M > 64: split-K only when the tile set cannot fill the SMs (plan_tiles)
  const TilePlan pl = plan_tiles((M + BLOCK_M - 1) / BLOCK_M, N, static_cast<int>((K + BLOCK_K - 1) / BLOCK_K), true, M);
  if (pl.splits <= 1) return 0;
  return static_cast<size_t>(pl.splits) * static_cast<size_t>(M) * static_cast<size_t>(N) * sizeof(float);
}

extern "C" int vb200_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* out,
                               int64_t ldo, int64_t M, int64_t N, int64_t K,
                               const vb_epilogue* epi, void* workspace, size_t workspace_bytes,
                               cudaStream_t stream) {
  VB_CHECK_ARG(A && W && out && epi);
  VB_CHECK_ARG(M > 0 && N > 0 && K > 0);
  VB_CHECK_ARG((lda % 8) == 0 && (ldw % 8) == 0 && lda >= K && ldw >= K);
  VB_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0);
  if (int r = validate_epi(epi, N)) return r;
  if (M <= 16) return vb_launch_gemv(A, lda, W, ldw, out, ldo, M, N, K, epi, stream);
  VB_CHECK_ARG(epi->rms_eps <= 0.f || epi->rowscale != nullptr);  // in-kernel rstd exists for M <= 16 only
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.num_k_blocks = static_cast<int>((K + BLOCK_K - 1) / BLOCK_K);
  p.a_mode = 0;
  p.a_box_bytes = BLOCK_M * BLOCK_K * 2;
  set_epilogue(p, epi);
  p.out = out;
  p.ldo = ldo;

  CUtensorMap ta, tb;
  const uint32_t estr2[2] = {1, 1};
  if (use_swap(M, N, K)) {
    // small M, long weight stream: kernel-M = N (weight rows), kernel-N = M (tokens); partials -> workspace -> reduce
    const int bn = M <= 32 ? 32 : 64;
    const int splits = swap_splits(M, N, K);
    const size_t need = static_cast<size_t>(splits) * M * N * sizeof(float);
    if (workspace == nullptr || workspace_bytes < need || !aligned16(workspace)) return VB_ERR_WORKSPACE;
    p.M = static_cast<int>(N);
    p.N = static_cast<int>(M);
    p.m_blocks = static_cast<int>((N + BLOCK_M - 1) / BLOCK_M);
    p.n_blocks = 1;
    p.splits = splits;
    p.swap = 1;
    p.ws = reinterpret_cast<float*>(workspace);
    p.ws_ld = N;
    p.ws_split_stride = M * N;
    uint64_t dA[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
    uint64_t sA[1] = {static_cast<uint64_t>(ldw) * 2};
    uint32_t bA[2] = {BLOCK_K, BLOCK_M};
    if (int r = make_tmap(&ta, W, 2, dA, sA, bA, estr2)) return r;
    uint64_t dB[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
    uint64_t sB[1] = {static_cast<uint64_t>(lda) * 2};
    uint32_t bB[2] = {BLOCK_K, static_cast<uint32_t>(bn)};
    if (int r = make_tmap(&tb, A, 2, dB, sB, bB, estr2)) return r;
    return launch_gemm_v2(bn, F_WS, ta, tb, p, stream);
  }

  p.M = static_cast<int>(M);
  p.N = static_cast<int>(N);
  p.m_blocks = static_cast<int>((M + BLOCK_M - 1) / BLOCK_M);
  uint64_t dA[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
  uint64_t sA[1] = {static_cast<uint64_t>(lda) * 2};
  uint32_t bA[2] = {BLOCK_K, BLOCK_M};
  if (int r = make_tmap(&ta, A, 2, dA, sA, bA, estr2)) return r;
  uint64_t dB[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
  uint64_t sB[1] = {static_cast<uint64_t>(ldw) * 2};
  if (const int rbn = resb_tile(M, N, p.num_k_blocks, v2_need(epi, 1))) {
    p.n_blocks = static_cast<int>((N + rbn - 1) / rbn);
    p.splits = 1;
    uint32_t bB[2] = {BLOCK_K, static_cast<uint32_t>(rbn)};
    if (int r = make_tmap(&tb, W, 2, dB, sB, bB, estr2)) return r;
    const int r = launch_gemm_v2_resb(rbn, v2_need(epi, 1), ta, tb, p, stream);
    if (r != VB_ERR_UNSUPPORTED) return r;
  }
  TilePlan pl = plan_tiles(p.m_blocks, N, p.num_k_blocks, true, M);
  if (pl.splits > 1) {
    const size_t need_ws = static_cast<size_t>(pl.splits) * M * N * sizeof(float);
    if (workspace == nullptr || workspace_bytes < need_ws || !aligned16(workspace)) pl = plan_tiles(p.m_blocks, N, p.num_k_blocks, false, M);
  }
  p.n_blocks = static_cast<int>((N + pl.bn - 1) / pl.bn);
  p.splits = pl.splits;
  if (pl.splits > 1) {
    p.ws = reinterpret_cast<float*>(workspace);
    p.ws_ld = N;
    p.ws_split_stride = M * N;
  }
  uint32_t bB[2] = {BLOCK_K, static_cast<uint32_t>(pl.bn)};
  if (int r = make_tmap(&tb, W, 2, dB, sB, bB, estr2)) return r;
  return launch_gemm_v2(pl.bn, v2_need(epi, pl.splits), ta, tb, p, stream);
}

static void conv_out_dims(int64_t h, int64_t w, int kh, int kw, int stride, int pad_h, int pad_w, int& ho, int& wo) {
  ho = static_cast<int>((h + 2 * pad_h - kh) / stride + 1);
  wo = static_cast<int>((w + 2 * pad_w - kw) / stride + 1);
}

extern "C" size_t vb200_conv_nhwc_workspace_size(int64_t nb, int64_t h, int64_t w, int64_t cin, int64_t cout, int kh,
                                                 int kw, int stride, int pad_h, int pad_w) {
  // split-K partials for convolutions whose pixel tiles cannot fill the SMs (0 for every other shape)
  if (nb <= 0 || h <= 0 || w <= 0 || cin <= 0 || cout <= 0 || kh <= 0 || kw <= 0 || (stride != 1 && stride != 2)) return 0;
  int ho, wo;
  conv_out_dims(h, w, kh, kw, stride, pad_h, pad_w, ho, wo);
  if (ho <= 0 || wo <= 0) return 0;
  int tw, th, tn;
  conv_pixel_tile(wo, ho, nb, tw, th, tn);
  const long long mb = static_cast<long long>((wo + tw - 1) / tw) * ((ho + th - 1) / th) * ((nb + tn - 1) / tn);
  const int kblocks = kh * kw * static_cast<int>((cin + BLOCK_K - 1) / BLOCK_K);
  const long long rows = nb * ho * wo;
  const TilePlan pl = plan_tiles(mb, cout, kblocks, true, rows);
  if (pl.splits <= 1) return 0;
  return static_cast<size_t>(pl.splits) * rows * cout * sizeof(float);
}

extern "C" int vb200_conv_nhwc_bf16(const void* X, const void* Wt, void* out, int64_t nb,
                                    int64_t h, int64_t w, int64_t cin, int64_t cout, int kh,
                                    int kw, int stride, int pad_h, int pad_w,
                                    const vb_epilogue* epi, void* workspace, size_t workspace_bytes,
                                    cudaStream_t stream) {
  // X [nb, h, w, cin] bf16 NHWC; Wt [cout, kh*kw, cin_pad] bf16 with cin_pad = ceil64(cin)
  // (zero padded); out [nb, ho, wo, cout(/2 if GLU)].
  VB_CHECK_ARG(X && Wt && out && epi);
  VB_CHECK_ARG(nb > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && kh > 0 && kw > 0);
  VB_CHECK_ARG(stride == 1 || stride == 2);
  VB_CHECK_ARG((cin % 8) == 0);
  if (int r = validate_epi(epi, cout)) return r;
  int ho, wo;
  conv_out_dims(h, w, kh, kw, stride, pad_h, pad_w, ho, wo);
  VB_CHECK_ARG(ho > 0 && wo > 0);
  const int cin_chunks = static_cast<int>((cin + BLOCK_K - 1) / BLOCK_K);
  const int cin_pad = cin_chunks * BLOCK_K;

  GemmParams p;
  memset(&p, 0, sizeof(p));
  int tw, th, tn;
  conv_pixel_tile(wo, ho, nb, tw, th, tn);
  p.a_mode = 1;
  p.cin_chunks = cin_chunks;
  p.kw = kw;
  p.stride = stride;
  p.pad_h = pad_h;
  p.pad_w = pad_w;
  p.tw = tw; p.th = th; p.tn = tn;
  p.wo = wo; p.ho = ho; p.nb = static_cast<int>(nb);
  p.tiles_w = (wo + tw - 1) / tw;
  p.tiles_h = (ho + th - 1) / th;
  const int tiles_n = static_cast<int>((nb + tn - 1) / tn);
  p.m_blocks = p.tiles_w * p.tiles_h * tiles_n;
  p.M = static_cast<int>(nb) * ho * wo;
  p.N = static_cast<int>(cout);
  p.num_k_blocks = kh * kw * cin_chunks;
  p.a_box_bytes = static_cast<uint32_t>(tw * th * tn) * BLOCK_K * 2;
  set_epilogue(p, epi);
  p.out = out;
  p.ldo = epi->glu != VB_GLU_NONE ? cout / 2 : cout;

  TilePlan pl = plan_tiles(p.m_blocks, cout, p.num_k_blocks, true, p.M);
  if (pl.splits > 1) {
    const size_t need_ws = static_cast<size_t>(pl.splits) * p.M * cout * sizeof(float);
    if (workspace == nullptr || workspace_bytes < need_ws || !aligned16(workspace)) pl = plan_tiles(p.m_blocks, cout, p.num_k_blocks, false, p.M);
  }
  p.splits = pl.splits;
  if (pl.splits > 1) {
    p.ws = reinterpret_cast<float*>(workspace);
    p.ws_ld = cout;
    p.ws_split_stride = static_cast<long long>(p.M) * cout;
  }
  p.n_blocks = static_cast<int>((cout + pl.bn - 1) / pl.bn);

  CUtensorMap ta, tb;
  uint64_t dA[4] = {static_cast<uint64_t>(cin), static_cast<uint64_t>(w), static_cast<uint64_t>(h),
                    static_cast<uint64_t>(nb)};
  uint64_t sA[3] = {static_cast<uint64_t>(cin) * 2, static_cast<uint64_t>(cin) * w * 2,
                    static_cast<uint64_t>(cin) * w * h * 2};
  // box extents are in traversed global elements: (tw-1)*stride+1 columns yield tw samples
  uint32_t bA[4] = {BLOCK_K, static_cast<uint32_t>((tw - 1) * stride + 1),
                    static_cast<uint32_t>((th - 1) * stride + 1), static_cast<uint32_t>(tn)};
  uint32_t eA[4] = {1, static_cast<uint32_t>(stride), static_cast<uint32_t>(stride), 1};
  if (int r = make_tmap(&ta, X, 4, dA, sA, bA, eA)) return r;
  uint64_t dB[2] = {static_cast<uint64_t>(kh) * kw * cin_pad, static_cast<uint64_t>(cout)};
  uint64_t sB[1] = {static_cast<uint64_t>(kh) * kw * cin_pad * 2};
  uint32_t bB[2] = {BLOCK_K, static_cast<uint32_t>(pl.bn)};
  const uint32_t estr2[2] = {1, 1};
  if (int r = make_tmap(&tb, Wt, 2, dB, sB, bB, estr2)) return r;
  return launch_gemm_v2(pl.bn, v2_need(epi, p.splits), ta, tb, p, stream);
}
