// vitron_b200 — LLaMA (Vicuna-7B) token-path kernels: RoPE + paged-KV append, paged decode
// attention (split-KV), multimodal embedding splice, greedy argmax. All HBM-bound.
//
// Reference arithmetic: HF transformers 4.31 LlamaAttention (rotate_half RoPE, fp32 softmax;
// restated in vitron/train/llama_flash_attn_monkey_patch.py:30-66), KV grown by torch.cat there —
// here a paged cache [num_pages, n_heads, page_size, head_dim]; splice =
// LlavaMetaForCausalLM.prepare_inputs_labels_for_multimodal (vitron/model/llava_arch.py:478-521).
#include "common.cuh"
#include <cstdlib>
#include "vitron_b200.h"
#include <limits.h>

namespace vb {

// ------------------------------------------------------------------ RoPE + KV append
// qkv row = [q(H*hd) | k(H*hd) | v(H*hd)]; one CTA per token, one thread per (head, 8-dim chunk).
__global__ void rope_kv_append_kernel(bf16* __restrict__ qkv, long long ld, const int32_t* __restrict__ positions,
                                      const int32_t* __restrict__ batch_of_token,
                                      const int32_t* __restrict__ slot_of_token, bf16* __restrict__ k_pages,
                                      bf16* __restrict__ v_pages, const int32_t* __restrict__ block_table,
                                      int max_pages, int H, int hd, int page_size, float log2_theta) {
  const long long tok = blockIdx.x;
  const int half = hd / 2;
  const int chunks = half / 8;  // 16-byte chunks per half head
  const int pos = positions[tok];
  const int slot = slot_of_token ? slot_of_token[tok] : pos;
  const int b = batch_of_token ? batch_of_token[tok] : 0;
  bf16* row = qkv + tok * ld;
  long long cache_off = -1;
  if (slot >= 0 && k_pages != nullptr && slot / page_size < max_pages) {  // a slot beyond the table is never written
    const int page = block_table[static_cast<long long>(b) * max_pages + slot / page_size];
    cache_off = (static_cast<long long>(page) * H) * page_size * hd + static_cast<long long>(slot % page_size) * hd;
  }
  for (int item = threadIdx.x; item < H * chunks; item += blockDim.x) {
    const int h = item / chunks, c = (item % chunks) * 8;
    float cs[8], sn[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float inv_freq = exp2f(-(2.0f * (c + j) / hd) * log2_theta);
      sincosf(static_cast<float>(pos) * inv_freq, &sn[j], &cs[j]);
    }
#pragma unroll
    for (int which = 0; which < 2; ++which) {  // 0: q, 1: k
      bf16* base = row + static_cast<long long>(which) * H * hd + h * hd;
      uint4 lo = *reinterpret_cast<const uint4*>(base + c);
      uint4 hi = *reinterpret_cast<const uint4*>(base + half + c);
      const uint32_t l4[4] = {lo.x, lo.y, lo.z, lo.w}, h4[4] = {hi.x, hi.y, hi.z, hi.w};
      uint32_t ol[4], oh[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 a = unpack_bf16(l4[j]), bb = unpack_bf16(h4[j]);
        // rotate_half: out_lo = x_lo*cos - x_hi*sin ; out_hi = x_hi*cos + x_lo*sin
        ol[j] = pack_bf16(a.x * cs[2 * j] - bb.x * sn[2 * j], a.y * cs[2 * j + 1] - bb.y * sn[2 * j + 1]);
        oh[j] = pack_bf16(bb.x * cs[2 * j] + a.x * sn[2 * j], bb.y * cs[2 * j + 1] + a.y * sn[2 * j + 1]);
      }
      const uint4 vlo = make_uint4(ol[0], ol[1], ol[2], ol[3]), vhi = make_uint4(oh[0], oh[1], oh[2], oh[3]);
      *reinterpret_cast<uint4*>(base + c) = vlo;
      *reinterpret_cast<uint4*>(base + half + c) = vhi;
      if (which == 1 && cache_off >= 0) {
        bf16* kc = k_pages + cache_off + static_cast<long long>(h) * page_size * hd;
        *reinterpret_cast<uint4*>(kc + c) = vlo;
        *reinterpret_cast<uint4*>(kc + half + c) = vhi;
      }
    }
    if (cache_off >= 0) {
      const bf16* vsrc = row + 2LL * H * hd + h * hd;
      bf16* vc = v_pages + cache_off + static_cast<long long>(h) * page_size * hd;
      *reinterpret_cast<uint4*>(vc + c) = *reinterpret_cast<const uint4*>(vsrc + c);
      *reinterpret_cast<uint4*>(vc + half + c) = *reinterpret_cast<const uint4*>(vsrc + half + c);
    }
  }
}

// ------------------------------------------------------------------ paged decode attention
// grid (splits, H, B); 4 warps; 8 lanes per key (16 dims each, head_dim 128), 2 keys in flight
// per lane group; every lane group runs its own online softmax, merged through smem at the end.
constexpr int DEC_THREADS = 128;
constexpr int DEC_CHUNK = 512;  // keys per split

// rotate_half RoPE of the 16 dims [16*sub, 16*sub+16) held by lane `sub` of an 8-lane group; the partner
// dims (+-64) live in lane sub^4. x is rounded to bf16 afterwards, like the unfused rope kernel.
// cs_table: [64 cos | 64 sin] of this sequence's position (vb200_rope_table), fp32
__device__ __forceinline__ void rope16(float (&x)[16], int sub, const float* __restrict__ cs_table) {
  const float4* c4 = reinterpret_cast<const float4*>(cs_table + (sub & 3) * 16);
  const float4* s4 = reinterpret_cast<const float4*>(cs_table + 64 + (sub & 3) * 16);
  float cs[16], sn[16];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 c = __ldg(c4 + j), s = __ldg(s4 + j);
    cs[4 * j] = c.x; cs[4 * j + 1] = c.y; cs[4 * j + 2] = c.z; cs[4 * j + 3] = c.w;
    sn[4 * j] = s.x; sn[4 * j + 1] = s.y; sn[4 * j + 2] = s.z; sn[4 * j + 3] = s.w;
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float partner = __shfl_xor_sync(0xffffffffu, x[j], 4);
    const float r = (sub < 4) ? x[j] * cs[j] - partner * sn[j] : x[j] * cs[j] + partner * sn[j];
    x[j] = __bfloat162float(__float2bfloat16(r));
  }
}

// table[b] = [cos(pos_b * f_i) | sin(pos_b * f_i)], i < hd/2, f_i = theta^(-2i/hd): shared by every head,
// split and layer of a decode step, so the transcendental work is done once per token.
__global__ void rope_table_kernel(const int32_t* __restrict__ positions, float* __restrict__ table, int half,
                                  float log2_theta) {
  const int b = blockIdx.x, i = threadIdx.x;
  pdl_trigger();
  pdl_wait();
  if (i >= half) return;
  const float inv_freq = exp2f(-(static_cast<float>(i) / half) * log2_theta);
  float sn, cs;
  sincosf(static_cast<float>(positions[b]) * inv_freq, &sn, &cs);
  table[b * 2 * half + i] = cs;
  table[b * 2 * half + half + i] = sn;
}

// BEAM: key j >= gen_start[b] of row b is read from the pages of row beam_src[b * src_ld + j] (through that row's block
// table): the beams of a request share their history without copying it. Keys below gen_start use the row's own table.
template <bool ROPE, int MAX_TRIPS, bool BEAM = false>
__global__ void __launch_bounds__(DEC_THREADS, 4)   // 4 CTAs per SM: the one-wave split policy counts on 4 x (SM count) slots
attn_decode_kernel(const bf16* __restrict__ q, long long ld_q, bf16* __restrict__ k_pages,
                   bf16* __restrict__ v_pages, const int32_t* __restrict__ block_table, int max_pages,
                   const int32_t* __restrict__ kv_len, int H, int page_size, float scale, int splits, int per,
                   float* __restrict__ ws_ml, float* __restrict__ ws_o, int* __restrict__ counters,
                   bf16* __restrict__ out, long long ld_o, const float* __restrict__ rope_table,
                   const int32_t* __restrict__ beam_src, int src_ld, const int32_t* __restrict__ gen_start) {
  // page_size == 64 and per % 64 == 0 (host-checked): a 64-key trip is exactly one page, and the page ids of
  // this split depend only on (split, per), so they are fetched before anything else (the block table is
  // constant during decoding -> safe ahead of the PDL dependency wait).
  constexpr int HD = 128;
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = lane >> 3, sub = lane & 7;
  const int32_t* bt = block_table + static_cast<long long>(b) * max_pages;
  const int c0 = split * per;
  int pg[MAX_TRIPS];
#pragma unroll
  for (int i = 0; i < MAX_TRIPS; ++i) {
    const int pi = c0 / 64 + i;
    pg[i] = (pi < max_pages && i * 64 < per) ? bt[pi] : 0;
  }
  // L2 prefetch of this CTA's first two pages (K and V, 16 KB each for this head) while the predecessor (the qkv projection,
  // which does not touch the cache) drains: pages of earlier tokens are constant during the step. One 128-byte line per
  // 4 lanes. The loop itself prefetches nothing: a prefetch two pages ahead from all 512 CTAs of the B = 8 step held ~48 MB
  // of lines in the 50 MB L2 until their use; without it a launch in the graphed step takes 52.5 instead of 62 us (H100 SXM,
  // 700 W).
  const long long pf_head = static_cast<long long>(h) * page_size * HD;
  const long long pf_stride = static_cast<long long>(H) * page_size * HD;
  auto prefetch_page = [&](int page) {
    const long long base = static_cast<long long>(page) * pf_stride + pf_head + static_cast<long long>(threadIdx.x) * 64;  // 128 thr x 128 B
    asm volatile("prefetch.global.L2 [%0];" ::"l"(k_pages + base));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(v_pages + base));
  };
  if (per > 0) prefetch_page(pg[0]);
  if (MAX_TRIPS > 1 && per > 64) prefetch_page(pg[1]);
  pdl_wait();
  // Dependents are released only now, after this grid's own dependency wait: released at kernel entry, the o-projection
  // GEMM and its split-K reduce (which rewrite the shared GEMM workspace and the hidden state) were let in while the qkv
  // projection that feeds this kernel was still in flight, and decode steps at batch >= 17 (GEMM, not GEMV, path) gave
  // different tokens from run to run.
  pdl_trigger();
  const int len = kv_len[b];
  const int c1 = min(len, c0 + per);
  const int gstart = BEAM ? gen_start[b] : 0;

  float qv[16];
  {
    const bf16* qp = q + static_cast<long long>(b) * ld_q + h * HD + sub * 16;
    uint4 u0 = *reinterpret_cast<const uint4*>(qp), u1 = *reinterpret_cast<const uint4*>(qp + 8);
    const uint32_t uu[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) { float2 f = unpack_bf16(uu[j]); qv[2 * j] = f.x; qv[2 * j + 1] = f.y; }
  }
  if (ROPE) {
    const float* cs_table = rope_table + b * HD;
    rope16(qv, sub, cs_table);
    // the split that owns the newest token (slot len-1) rotates k, and appends k / v to their page
    const int tnew = len - 1;
    if (tnew >= c0 && tnew < c1) {
      if (warp == 0) {  // whole warp runs the shuffles; lane group 0 stores
        float kv_[16];
        const bf16* kp = q + static_cast<long long>(b) * ld_q + (static_cast<long long>(H) + h) * HD + sub * 16;
        uint4 u0 = *reinterpret_cast<const uint4*>(kp), u1 = *reinterpret_cast<const uint4*>(kp + 8);
        const uint32_t uu[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) { float2 f = unpack_bf16(uu[j]); kv_[2 * j] = f.x; kv_[2 * j + 1] = f.y; }
        rope16(kv_, sub, cs_table);
        if (grp == 0) {
          const long long off = static_cast<long long>(bt[tnew / page_size]) * H * page_size * HD +
                                static_cast<long long>(h) * page_size * HD + static_cast<long long>(tnew % page_size) * HD + sub * 16;
          uint32_t w[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) w[j] = pack_bf16(kv_[2 * j], kv_[2 * j + 1]);
          *reinterpret_cast<uint4*>(k_pages + off) = make_uint4(w[0], w[1], w[2], w[3]);
          *reinterpret_cast<uint4*>(k_pages + off + 8) = make_uint4(w[4], w[5], w[6], w[7]);
          const bf16* vp = q + static_cast<long long>(b) * ld_q + (2LL * H + h) * HD + sub * 16;
          *reinterpret_cast<uint4*>(v_pages + off) = *reinterpret_cast<const uint4*>(vp);
          *reinterpret_cast<uint4*>(v_pages + off + 8) = *reinterpret_cast<const uint4*>(vp + 8);
        }
      }
      __threadfence_block();
      __syncthreads();
    }
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) qv[j] *= scale;
  float m = -INFINITY, l = 0.f, o[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) o[j] = 0.f;
  const long long head_off = static_cast<long long>(h) * page_size * HD + sub * 16;
  const long long page_stride = static_cast<long long>(H) * page_size * HD;

  // 16 lane groups per CTA. The split is walked in HALF pages of 32 keys: lane group gid takes the keys gid and gid + 16 of
  // the half (2 K rows + 2 V rows = 128 B per lane) and the loop is software pipelined over two register buffers — the
  // loads of half h + 1 are issued BEFORE the dot products / softmax / PV of half h, so every warp has loads in flight all
  // the time (ncu of the one-buffer version: 4.7 long-scoreboard stall cycles per issued instruction, issue slots 33 % busy,
  // DRAM traffic = algorithmic: the kernel waited, it did not waste). Same register footprint as 4 keys per 64-key trip.
  const int gid = warp * 4 + grp;
  struct Half { uint4 k[2][2], v[2][2]; };
  const int nh = c1 > c0 ? (c1 - c0 + 31) / 32 : 0;   // halves this split holds (warp-uniform)
  auto load_half = [&](int hs, Half& h) {
    const long long pbase = static_cast<long long>(pg[hs >> 1]) * page_stride + head_off;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int kk = gid + 16 * u + 32 * (hs & 1);  // key inside the page
      const bool has = c0 + 64 * (hs >> 1) + kk < c1;
      long long off = pbase + static_cast<long long>(has ? kk : 0) * HD;
      if (BEAM) {
        const int key = c0 + 64 * (hs >> 1) + kk;
        if (has && key >= gstart) {
          const int src_row = beam_src[static_cast<long long>(b) * src_ld + key];
          off = static_cast<long long>(block_table[static_cast<long long>(src_row) * max_pages + key / 64]) * page_stride +
                head_off + static_cast<long long>(kk) * HD;
        }
      }
      h.k[u][0] = *reinterpret_cast<const uint4*>(k_pages + off);
      h.k[u][1] = *reinterpret_cast<const uint4*>(k_pages + off + 8);
      h.v[u][0] = *reinterpret_cast<const uint4*>(v_pages + off);
      h.v[u][1] = *reinterpret_cast<const uint4*>(v_pages + off + 8);
    }
  };
  auto compute_half = [&](int hs, const Half& h) {
    float sc[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const uint32_t kw[8] = {h.k[u][0].x, h.k[u][0].y, h.k[u][0].z, h.k[u][0].w, h.k[u][1].x, h.k[u][1].y, h.k[u][1].z, h.k[u][1].w};
      float a = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float2 f = unpack_bf16(kw[j]);
        a += qv[2 * j] * f.x + qv[2 * j + 1] * f.y;
      }
      sc[u] = a;
    }
#pragma unroll
    for (int sh = 1; sh < 8; sh <<= 1) {
#pragma unroll
      for (int u = 0; u < 2; ++u) sc[u] += __shfl_xor_sync(0xffffffffu, sc[u], sh);
    }
    float mn = m;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const bool has = c0 + 64 * (hs >> 1) + gid + 16 * u + 32 * (hs & 1) < c1;
      if (!has) sc[u] = -INFINITY;
      mn = fmaxf(mn, sc[u]);
    }
    const float msafe = (mn == -INFINITY) ? 0.f : mn;
    const float corr = __expf(m - msafe);  // m = -inf on first use -> 0
    float pr[2];
    float psum = 0.f;
#pragma unroll
    for (int u = 0; u < 2; ++u) { pr[u] = __expf(sc[u] - msafe); psum += pr[u]; }
    l = l * corr + psum;
    m = mn;
#pragma unroll
    for (int j = 0; j < 16; ++j) o[j] *= corr;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const uint32_t vw[8] = {h.v[u][0].x, h.v[u][0].y, h.v[u][0].z, h.v[u][0].w, h.v[u][1].x, h.v[u][1].y, h.v[u][1].z, h.v[u][1].w};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float2 f = unpack_bf16(vw[j]);
        o[2 * j] += pr[u] * f.x;
        o[2 * j + 1] += pr[u] * f.y;
      }
    }
  };
  Half buf0, buf1;
  if (nh > 0) load_half(0, buf0);
#pragma unroll
  for (int hs = 0; hs < 2 * MAX_TRIPS; hs += 2) {   // one iteration = one 64-key page
    if (hs >= nh) break;                            // warp-uniform (the shuffles use the full mask)
    if (hs + 1 < nh) load_half(hs + 1, buf1);
    compute_half(hs, buf0);
    if (hs + 1 >= nh) break;
    if (hs + 2 < nh && hs + 2 < 2 * MAX_TRIPS) load_half(hs + 2, buf0);
    compute_half(hs + 1, buf1);
  }

  // ---- merge the 16 lane groups
  __shared__ float sm_m[16], sm_l[16];
  __shared__ float sm_o[16][HD + 4];
  if (sub == 0) { sm_m[gid] = m; sm_l[gid] = l; }
#pragma unroll
  for (int j = 0; j < 16; ++j) sm_o[gid][sub * 16 + j] = o[j];
  __syncthreads();
  const int d = threadIdx.x;  // one thread per output dim
  float M = -INFINITY;
#pragma unroll
  for (int g = 0; g < 16; ++g) M = fmaxf(M, sm_m[g]);
  float L = 0.f, O = 0.f;
#pragma unroll
  for (int g = 0; g < 16; ++g) {
    const float w = (sm_m[g] == -INFINITY) ? 0.f : __expf(sm_m[g] - M);
    L += sm_l[g] * w;
    O += sm_o[g][d] * w;
  }
  if (splits == 1) {
    out[static_cast<long long>(b) * ld_o + h * HD + d] = __float2bfloat16(L > 0.f ? O / L : 0.f);
  } else {
    const long long base = (static_cast<long long>(b) * H + h) * splits;
    const long long idx = base + split;
    if (d == 0) { ws_ml[idx * 2] = M; ws_ml[idx * 2 + 1] = L; }
    ws_o[idx * HD + d] = O;
    // the CTA that finishes this (batch, head) last merges the split partials (fixed order)
    __shared__ int is_last;
    __threadfence();
    __syncthreads();
    if (d == 0) is_last = (atomicAdd(&counters[b * H + h], 1) == splits - 1) ? 1 : 0;
    __syncthreads();
    if (is_last) {
      __threadfence();
      float Mx = -INFINITY;
      for (int s = 0; s < splits; ++s) Mx = fmaxf(Mx, __ldcg(&ws_ml[(base + s) * 2]));
      float Ls = 0.f, Os = 0.f;
      for (int s = 0; s < splits; ++s) {
        const float ms = __ldcg(&ws_ml[(base + s) * 2]);
        const float w = (ms == -INFINITY) ? 0.f : __expf(ms - Mx);
        Ls += __ldcg(&ws_ml[(base + s) * 2 + 1]) * w;
        Os += __ldcg(&ws_o[(base + s) * HD + d]) * w;
      }
      out[static_cast<long long>(b) * ld_o + h * HD + d] = __float2bfloat16(Ls > 0.f ? Os / Ls : 0.f);
      if (d == 0) counters[b * H + h] = 0;
    }
  }
}

// ------------------------------------------------------------------ multimodal splice
__global__ void splice_kernel(const bf16* __restrict__ embed, long long vocab, const bf16* __restrict__ feats,
                              long long n_feat, const int32_t* __restrict__ srcmap, bf16* __restrict__ out,
                              int d) {
  const long long row = blockIdx.x;
  pdl_trigger();
  pdl_wait();
  const int src = srcmap[row];
  const bf16* sp = nullptr;
  if (src >= 0 && src < vocab) sp = embed + static_cast<long long>(src) * d;
  else if (src < 0 && src != INT_MIN && -(static_cast<long long>(src) + 1) < n_feat)
    sp = feats + (-(static_cast<long long>(src) + 1)) * d;
  uint4* dst = reinterpret_cast<uint4*>(out + row * d);
  const int nvec = d / 8;
  if (sp) {
    const uint4* s4 = reinterpret_cast<const uint4*>(sp);
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) dst[i] = s4[i];
  } else {
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) dst[i] = make_uint4(0, 0, 0, 0);
  }
}

// ------------------------------------------------------------------ argmax (first maximal index)
template <typename T>
__global__ void __launch_bounds__(1024) argmax_kernel(const T* __restrict__ x, long long ld, int n, int64_t* __restrict__ out) {
  __shared__ float sv[32];
  __shared__ int si[32];
  const T* row = x + blockIdx.x * ld;
  float best = -INFINITY;
  int bi = INT_MAX;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float v = static_cast<float>(row[i]);
    if (v > best || (bi == INT_MAX && v == v)) { best = v; bi = i; }  // NaNs never win
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x < 32) {
    best = threadIdx.x < (blockDim.x >> 5) ? sv[threadIdx.x] : -INFINITY;
    bi = threadIdx.x < (blockDim.x >> 5) ? si[threadIdx.x] : INT_MAX;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best, o);
      int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (threadIdx.x == 0) out[blockIdx.x] = bi == INT_MAX ? 0 : bi;
  }
}

// greedy decode bookkeeping fused with the arg-max: one CTA per sequence
__global__ void __launch_bounds__(1024)
argmax_advance_kernel(const float* __restrict__ logits, long long ld, int n, int64_t* __restrict__ out_idx,
                      int32_t* __restrict__ next_src, int32_t* __restrict__ positions, int32_t* __restrict__ kv_len,
                      int64_t* __restrict__ token_log, int log_stride, const int32_t* __restrict__ prompt_len) {
  __shared__ float sv[32];
  __shared__ int si[32];
  const int b = blockIdx.x;
  pdl_trigger();
  pdl_wait();
  const float* row = logits + b * ld;
  float best = -INFINITY;
  int bi = INT_MAX;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float v = row[i];
    if (v > best || (bi == INT_MAX && v == v)) { best = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x < 32) {
    best = sv[threadIdx.x];
    bi = si[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best, o);
      int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (threadIdx.x == 0) {
      if (bi == INT_MAX) bi = 0;
      out_idx[b] = bi;
      if (next_src) next_src[b] = bi;
      if (token_log) {
        const int step = kv_len[b] - prompt_len[b];  // tokens generated before this one
        if (step >= 0 && step < log_stride) token_log[static_cast<long long>(b) * log_stride + step] = bi;
      }
      if (positions) positions[b] += 1;
      if (kv_len) kv_len[b] += 1;
    }
  }
}

// ------------------------------------------------------------------ sampling (temperature, top-k, top-p, Philox draw)
// One CTA per row; the row is staged in shared memory. Both cuts are radix selects over a 32-bit order key of the logit
// (11 + 11 + 10 bit digits): top-k by per-bin counts, top-p by per-bin mass. Masses are fixed point (p * 2^40, p <= 1) so
// every sum is an integer sum: the same logits give the same token on every run, whatever the order of the atomics.
constexpr int SMP_THREADS = 1024;
constexpr int SMP_BINS = 2048;
constexpr int SMP_MAX_N = 49152;               // 192 KB of staged row + 24 KB of histograms fit the 227 KB of an SM
constexpr float SMP_FIX = 1099511627776.0f;    // 2^40

// monotone map float -> uint32 (larger value, larger key); NaN -> 0, below every number (-inf -> 0x007fffff); -0 == +0
__device__ __forceinline__ uint32_t order_key(float v) {
  if (v != v) return 0u;
  const uint32_t u = v == 0.f ? 0u : __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Random123 philox4x32-10
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

template <typename T>
__device__ __forceinline__ T warp_inclusive_scan(T v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T x = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += x;
  }
  return v;
}

// exclusive prefix of v over threadIdx order (blockDim == 1024); *total gets the block sum. buf: 33 entries.
template <typename T>
__device__ T block_exclusive_scan(T v, T* buf, T* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T inc = warp_inclusive_scan(v);
  if (lane == 31) buf[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const T w = buf[lane];
    const T wi = warp_inclusive_scan(w);
    buf[lane] = wi - w;
    if (lane == 31) buf[32] = wi;
  }
  __syncthreads();
  const T r = buf[warp] + inc - v;
  *total = buf[32];
  __syncthreads();
  return r;
}

// Shared-memory scratch of the radix selects below (one CTA of SMP_THREADS threads).
struct SmpScratch {
  uint32_t* h_cnt;               // [SMP_BINS]
  unsigned long long* h_mass;    // [SMP_BINS]
  unsigned long long* s_u64;     // [33]
  uint32_t* s_bin;
  unsigned long long* s_above;
};

// p_i = exp(z_i - max z), z = v / T, as fixed point; the maximum itself is exactly 1 (also for +-inf)
__device__ __forceinline__ unsigned long long smp_mass(float v, float mx, float temp) {
  const float p = v == mx ? 1.f : expf((v - mx) / temp);
  return __float2ull_rn(p * SMP_FIX);
}

// 64-bit add to shared memory as two native 32-bit atomics, the low word's carry going to the high word: the 64-bit
// shared atomicAdd is a compare-and-swap loop, which a bin many entries fall into turns into long retry chains. The sum
// is exact, so the order of the adds does not matter.
__device__ __forceinline__ void smp_add_u64(unsigned long long* a, unsigned long long v) {
  uint32_t* w = reinterpret_cast<uint32_t*>(a);
  const uint32_t lo = static_cast<uint32_t>(v), hi = static_cast<uint32_t>(v >> 32);
  const uint32_t old = atomicAdd(w, lo);
  const uint32_t up = hi + (old + lo < old ? 1u : 0u);
  if (up) atomicAdd(w + 1, up);
}

// One radix level over the kept keys (order_key >= thr) of srow[0, n) whose bits above `shift + width` equal `prefix`:
// histogram of the digit, then the lowest non-empty bin whose "before" value (count / mass of the kept keys in strictly
// higher bins, plus `above`) is still below `limit`. Returns that bin; *s_above gets its "before" value.
__device__ uint32_t smp_radix_level(const float* srow, int n, uint32_t thr, float mx, float temp, const SmpScratch& sc,
                                    uint32_t prefix, uint32_t himask, int shift, uint32_t dmask, bool by_mass,
                                    unsigned long long above, unsigned long long limit) {
  const int tid = threadIdx.x;
  for (int i = tid; i < SMP_BINS; i += SMP_THREADS) { sc.h_cnt[i] = 0; sc.h_mass[i] = 0; }
  if (tid == 0) *sc.s_bin = SMP_BINS;
  __syncthreads();
  for (int i = tid; i < n; i += SMP_THREADS) {
    const float v = srow[i];
    const uint32_t key = order_key(v);
    if (key >= thr && (key & himask) == prefix) {
      const uint32_t d = (key >> shift) & dmask;
      atomicAdd(&sc.h_cnt[d], 1u);
      if (by_mass) smp_add_u64(&sc.h_mass[d], smp_mass(v, mx, temp));
    }
  }
  __syncthreads();
  // thread t owns bins hi = 2047 - 2t and hi - 1; scan in descending bin order
  const int hi = SMP_BINS - 1 - 2 * tid, lo = hi - 1;
  const unsigned long long w_hi = by_mass ? sc.h_mass[hi] : sc.h_cnt[hi], w_lo = by_mass ? sc.h_mass[lo] : sc.h_cnt[lo];
  unsigned long long tot;
  const unsigned long long before_hi = above + block_exclusive_scan(w_hi + w_lo, sc.s_u64, &tot);
  const unsigned long long before_lo = before_hi + w_hi;
  if (sc.h_cnt[lo] > 0 && before_lo < limit) atomicMin(sc.s_bin, static_cast<uint32_t>(lo));
  else if (sc.h_cnt[hi] > 0 && before_hi < limit) atomicMin(sc.s_bin, static_cast<uint32_t>(hi));
  __syncthreads();
  const uint32_t sel = *sc.s_bin;
  if (sel == static_cast<uint32_t>(lo)) *sc.s_above = before_lo;
  if (sel == static_cast<uint32_t>(hi)) *sc.s_above = before_hi;
  __syncthreads();
  return sel;
}

// the cut key: radix descent over the three digits (bits 31..21, 20..10, 9..0)
__device__ uint32_t smp_select_key(const float* srow, int n, uint32_t thr, float mx, float temp, const SmpScratch& sc,
                                   bool by_mass, unsigned long long limit) {
  uint32_t prefix = 0, himask = 0;
  unsigned long long above = 0;
#pragma unroll 1
  for (int lvl = 0; lvl < 3; ++lvl) {
    const int shift = lvl == 0 ? 21 : lvl == 1 ? 10 : 0;
    const uint32_t d = smp_radix_level(srow, n, thr, mx, temp, sc, prefix, himask, shift, lvl == 2 ? 1023u : 2047u,
                                       by_mass, above, limit);
    above = *sc.s_above;
    prefix |= d << shift;
    himask = lvl == 0 ? 0xFFE00000u : 0xFFFFFC00u;
  }
  return prefix;
}

__device__ unsigned long long smp_kept_mass(const float* srow, int n, uint32_t thr, float mx, float temp,
                                            const SmpScratch& sc) {
  unsigned long long m = 0, tot;
  for (int i = threadIdx.x; i < n; i += SMP_THREADS) {
    const float v = srow[i];
    if (order_key(v) >= thr) m += smp_mass(v, mx, temp);
  }
  block_exclusive_scan(m, sc.s_u64, &tot);
  return tot;
}

// The warpers of the staged row srow[0, n) (values v, z = v / temp, mx = max v, `valid` = non-NaN count). Returns thr:
// the kept set is {i : order_key(v_i) >= thr}; *total gets its mass.
//   top-k: the k-th largest kept key; ties at it stay (count of strictly larger keys < k);
//   top-p: keep i iff the kept mass of strictly larger keys is < top_p * total; the maximum always stays, and with
//   min_keep = 2 so does every key with fewer than 2 strictly larger kept keys (TopPLogitsWarper's min_tokens_to_keep).
__device__ uint32_t smp_warp(const float* srow, int n, uint32_t valid, float mx, float temp, int top_k, float top_p,
                             int min_keep, const SmpScratch& sc, unsigned long long* total) {
  uint32_t thr = 1u;   // thr = 1 drops only the NaNs
  if (top_k > 0 && static_cast<uint32_t>(top_k) < valid)
    thr = smp_select_key(srow, n, thr, mx, temp, sc, false, static_cast<unsigned long long>(top_k));
  *total = smp_kept_mass(srow, n, thr, mx, temp, sc);
  if (top_p < 1.f) {
    uint32_t cut;
    if (top_p <= 0.f) {
      cut = order_key(mx);
    } else {
      const unsigned long long limit =
          static_cast<unsigned long long>(ceil(static_cast<double>(top_p) * static_cast<double>(*total)));
      cut = smp_select_key(srow, n, thr, mx, temp, sc, true, limit);
    }
    if (min_keep > 1) cut = min(cut, smp_select_key(srow, n, thr, mx, temp, sc, false, min_keep));
    thr = cut;
    *total = smp_kept_mass(srow, n, thr, mx, temp, sc);
  }
  return thr;
}

__global__ void __launch_bounds__(SMP_THREADS, 1)
sample_advance_kernel(const float* __restrict__ logits, long long ld, int n, const vb_sample_params* __restrict__ prm,
                      int64_t* __restrict__ out_idx, int32_t* __restrict__ next_src, int32_t* __restrict__ positions,
                      int32_t* __restrict__ kv_len, int64_t* __restrict__ token_log, int log_stride,
                      const int32_t* __restrict__ prompt_len) {
  extern __shared__ float srow[];
  __shared__ uint32_t h_cnt[SMP_BINS];
  __shared__ unsigned long long h_mass[SMP_BINS];
  __shared__ unsigned long long s_u64[33];
  __shared__ uint32_t s_u32[33];
  __shared__ float s_f32[32];
  __shared__ uint32_t s_bin;
  __shared__ unsigned long long s_above;
  __shared__ int s_tok;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_wait();      // the logits and the decode state come from the predecessors
  pdl_trigger();
  const float* row = logits + b * ld;

  // ---- stage the row (rows of an odd-V matrix are only 4-byte aligned: scalar head, float4 body, scalar tail)
  float mx = -INFINITY;
  uint32_t valid = 0;
  auto take = [&](int i, float v) {
    srow[i] = v;
    if (v == v) { mx = fmaxf(mx, v); ++valid; }
  };
  int head = static_cast<int>(((16u - (reinterpret_cast<uintptr_t>(row) & 15u)) & 15u) >> 2);
  if (head > n) head = n;
  const int nvec = (n - head) >> 2;
  if (tid < head) take(tid, row[tid]);
  const float4* row4 = reinterpret_cast<const float4*>(row + head);
  for (int j = tid; j < nvec; j += SMP_THREADS) {
    const float4 v = row4[j];
    const int i = head + 4 * j;
    take(i, v.x); take(i + 1, v.y); take(i + 2, v.z); take(i + 3, v.w);
  }
  for (int i = head + 4 * nvec + tid; i < n; i += SMP_THREADS) take(i, row[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    valid += __shfl_xor_sync(0xffffffffu, valid, o);
  }
  if (lane == 0) { s_f32[warp] = mx; s_u32[warp] = valid; }
  __syncthreads();
  mx = s_f32[lane];
  valid = s_u32[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    valid += __shfl_xor_sync(0xffffffffu, valid, o);
  }
  __syncthreads();

  int tok = 0;   // a row without a number samples token 0, like the arg-max
  if (valid > 0) {
    const float temp = prm->temperature;
    const SmpScratch sc{h_cnt, h_mass, s_u64, &s_bin, &s_above};
    unsigned long long total;
    const uint32_t thr = smp_warp(srow, n, valid, mx, temp, prm->top_k, prm->top_p, 1, sc, &total);
    auto mass_of = [&](float v) { return smp_mass(v, mx, temp); };

    // draw: u = (philox[0] >> 8) * 2^-24; first kept index (vocabulary order) whose inclusive prefix mass > u * total.
    // prefix > u * total  <=>  prefix > floor(a * total / 2^24) for integer prefix, a = philox[0] >> 8
    const uint32_t t = (kv_len != nullptr && prompt_len != nullptr) ? static_cast<uint32_t>(kv_len[b] - prompt_len[b]) : 0u;
    const unsigned long long seed = prm->seed;
    const uint4 r = philox4x32_10(make_uint4(t, static_cast<uint32_t>(b), 0u, 0u), static_cast<uint32_t>(seed),
                                  static_cast<uint32_t>(seed >> 32));
    const unsigned long long a = r.x >> 8;
    const unsigned long long target = (__umul64hi(a, total) << 40) | ((a * total) >> 24);
    // thread t owns the contiguous chunk [t*C, t*C + C); the chunk sum is read rotated by t (conflict-free banks)
    const int C = (n + SMP_THREADS - 1) / SMP_THREADS;
    const int c0 = tid * C, c1 = min(n, c0 + C);
    unsigned long long m = 0;
    for (int j = 0; j < C; ++j) {
      const int i = c0 + (j + tid) % C;
      if (i < c1) {
        const float v = srow[i];
        if (order_key(v) >= thr) m += mass_of(v);
      }
    }
    unsigned long long tot;
    const unsigned long long before = block_exclusive_scan(m, s_u64, &tot);
    if (before <= target && target < before + m) {   // exactly one thread: target < total, the chunks partition it
      unsigned long long run = before;
      for (int i = c0; i < c1; ++i) {
        const float v = srow[i];
        if (order_key(v) < thr) continue;
        run += mass_of(v);
        if (run > target) { s_tok = i; break; }
      }
    }
    __syncthreads();
    tok = s_tok;
  }

  if (tid == 0) {
    if (out_idx) out_idx[b] = tok;
    if (next_src) next_src[b] = tok;
    if (token_log) {
      const int step = kv_len[b] - prompt_len[b];  // tokens generated before this one
      if (step >= 0 && step < log_stride) token_log[static_cast<long long>(b) * log_stride + step] = tok;
    }
    if (positions) positions[b] += 1;
    if (kv_len) kv_len[b] += 1;
  }
}

// ------------------------------------------------------------------ beam search step (HF 4.31 beam_search + BeamSearchScorer)
// One CTA per row r = b * k + j: log-softmax of the row and its top 2k candidates (score desc, then index asc) by repeated
// block arg-max, where only the thread that owned the last winner rescans its strided slice. The request's top 2k lie in
// the union of its rows' top 2k: the CTA that arrives last for request b ranks those k * 2k candidates, runs the scorer
// and does the bookkeeping of all k rows. Candidate order is total (flat index = j * n + token breaks every tie), so the
// result does not depend on arrival order.
constexpr int BM_THREADS = 1024;
constexpr int BM_MAX_K = 16;
constexpr int BM_MAX_N = 49152;              // 192 KB of staged row
constexpr int BM_STAGE = 256;                // beam-source columns staged per pass of the history reorder
constexpr size_t BM_COUNTER_BYTES = 16384;   // B <= 4096 arrival counters, then the candidates
constexpr int BM_SENTINEL = 0x40000000;      // flat index of a missing candidate (row with fewer than 2k entries)

__device__ __forceinline__ bool bm_better(float sa, int ia, float sb, int ib) {
  return sa > sb || (sa == sb && ia < ib);
}

// The history-reorder stage buffer. The sampling variant overlays the radix selects' mass histogram on it: the selects
// finish before the reorder starts, and the row (<= 192 KB) plus both would not fit an SM's shared memory.
template <bool SAMPLE>
struct BmStage {
  typedef int32_t type[BM_MAX_K][BM_STAGE];
  __device__ static type& get(type& s) { return s; }
};
template <>
struct BmStage<true> {
  union type {
    int32_t stage[BM_MAX_K][BM_STAGE];
    unsigned long long mass[SMP_BINS];
  };
  __device__ static int32_t (&get(type& s))[BM_MAX_K][BM_STAGE] { return s.stage; }
};

// The block-wide max and sum of the row log-softmax (BM_THREADS threads, s_f: 32 floats). The beam kernel and the logits
// processors' LOGPROBS mode share them, so that the log-probabilities the processors write are bit-identical to the ones
// the beam kernel computes itself.
__device__ __forceinline__ float bm_block_max(float mx, float* s_f, int lane, int warp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) s_f[warp] = mx;
  __syncthreads();
  mx = s_f[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  __syncthreads();
  return mx;
}

__device__ __forceinline__ float bm_block_sum(float sum, float* s_f, int lane, int warp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) s_f[warp] = sum;
  __syncthreads();
  sum = s_f[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  __syncthreads();
  return sum;
}

// Gumbel noise of flat index f of search b at step t: U = (2 * (x >> 9) + 1) * 2^-24 in (0, 1), x = word f % 4 of
// Philox4x32-10(counter (t, b, f / 4, 1), key (seed_lo, seed_hi)); the noise is -log(-log U).
__device__ __forceinline__ float bm_gumbel(uint32_t x) {
  const float u = static_cast<float>(2u * (x >> 9) + 1u) * 5.9604644775390625e-8f;   // 2^-24
  return -logf(-logf(u));
}

// SAMPLE = false: beam search. SAMPLE = true: beam sampling (HF 4.31 beam_sample): the rows' scores are warped
// (temperature, top-k, top-p with 2 kept) and 2k candidates per request are drawn without replacement as the top 2k of
// key = w + Gumbel noise; they are then ranked by warped score and go through the same scorer.
// LOGPROBS: the rows already hold (processed) log-probabilities, written by logits_process_kernel's LOGPROBS mode: the
// candidate score is row[i] + beam score, with no max / sum pass of its own (the warpers still cut on the row's max).
template <bool SAMPLE, bool LOGPROBS = false>
__global__ void __launch_bounds__(BM_THREADS, 1)
beam_advance_kernel(const float* __restrict__ logits, long long ld, int n, int k, const vb_beam_params* __restrict__ prm,
                    float* __restrict__ beam_score, int32_t* __restrict__ parent, int32_t* __restrict__ done,
                    int32_t* __restrict__ beam_src, int src_ld, double* __restrict__ hyp_score,
                    int32_t* __restrict__ hyp_len, int32_t* __restrict__ hyp_seq, int32_t* __restrict__ hyp_count,
                    int64_t* __restrict__ hyp_ids, int hyp_ld, int32_t* __restrict__ next_src,
                    int32_t* __restrict__ positions, int32_t* __restrict__ kv_len, int64_t* __restrict__ token_log,
                    int log_stride, const int32_t* __restrict__ prompt_len, float* __restrict__ cand_s,
                    int32_t* __restrict__ cand_i, int32_t* __restrict__ counters,
                    const vb_sample_params* __restrict__ sprm, float* __restrict__ cand_w) {
  extern __shared__ float srow[];
  __shared__ float s_f[32];
  __shared__ int s_i[32];
  __shared__ float s_ws;
  __shared__ int s_wi, s_last, s_t, s_P;
  __shared__ float m_s[BM_MAX_K * 2 * BM_MAX_K];
  __shared__ int m_i[BM_MAX_K * 2 * BM_MAX_K];
  __shared__ float t_s[2 * BM_MAX_K];
  __shared__ int t_i[2 * BM_MAX_K];
  __shared__ int c_par[BM_MAX_K], c_tok[BM_MAX_K], h_src[BM_MAX_K];
  __shared__ float c_sc[BM_MAX_K];
  __shared__ typename BmStage<SAMPLE>::type stage_buf;
  auto& stage = BmStage<SAMPLE>::get(stage_buf);
  const int r = blockIdx.x, b = r / k, j = r % k, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int k2 = 2 * k;
  pdl_wait();      // logits, scores and the decode state come from the predecessors
  pdl_trigger();

  // ---- log-softmax statistics of the row (NaN counts as -inf); fixed reduction order
  const float* row = logits + r * ld;
  float mx = -INFINITY;
  for (int i = tid; i < n; i += BM_THREADS) {
    float v = row[i];
    if (v != v) v = -INFINITY;
    srow[i] = v;
    mx = fmaxf(mx, v);
  }
  mx = bm_block_max(mx, s_f, lane, warp);
  float logz = 0.f;
  if constexpr (!LOGPROBS) {
    float sum = 0.f;
    if (mx > -INFINITY)
      for (int i = tid; i < n; i += BM_THREADS) sum += expf(srow[i] - mx);
    logz = logf(bm_block_sum(sum, s_f, lane, warp));
  }
  const float bsc = beam_score[r];
  // candidate score = log_softmax + beam score, as torch computes it: (x - max) - log(sum exp(x - max))
  auto score_of = [&](int i) -> float {
    if constexpr (LOGPROBS) return mx == -INFINITY ? -INFINITY : srow[i] + bsc;
    else return mx == -INFINITY ? -INFINITY : ((srow[i] - mx) - logz) + bsc;
  };
  // the row's log-probability from its logit as read from memory (warped scores are recomputed from it)
  auto lp_of = [&](int i) -> float {
    if constexpr (LOGPROBS) return row[i];
    else return (row[i] - mx) - logz;
  };
  float temp = 1.f;
  if constexpr (SAMPLE) {
    // ---- the warpers' kept set, cut on d = (x - max x) / T: within the row the warped scores w are d plus a constant,
    // and d spreads over the float exponents as the sampler's logits do (w of a flat row shares one exponent, and its
    // histogram atomics would all hit a few bins). Then srow[i] = w_i + Gumbel noise of (b, flat index) over the kept
    // entries with w > -inf, -inf elsewhere.
    __shared__ uint32_t h_cnt[SMP_BINS];
    __shared__ unsigned long long s_u64[33];
    __shared__ uint32_t s_bin;
    __shared__ unsigned long long s_above;
    temp = sprm->temperature;
    uint32_t thr = 0xFFFFFFFFu;   // a row without a number keeps nothing
    if (mx > -INFINITY) {
      for (int i = tid; i < n; i += BM_THREADS) srow[i] = (srow[i] - mx) / temp;
      __syncthreads();
      const SmpScratch sc{h_cnt, stage_buf.mass, s_u64, &s_bin, &s_above};
      const int top_k = sprm->top_k > 0 ? max(sprm->top_k, 2) : 0;
      unsigned long long total;
      thr = smp_warp(srow, n, static_cast<uint32_t>(n), 0.f, 1.f, top_k, sprm->top_p, 2, sc, &total);
    }
    const uint32_t t = static_cast<uint32_t>(kv_len[b * k] - prompt_len[b * k]);
    const unsigned long long seed = sprm->seed;
    const uint32_t f0 = static_cast<uint32_t>(j) * n, g0 = f0 >> 2, g1 = (f0 + n - 1) >> 2;
    for (uint32_t g = g0 + tid; g <= g1; g += BM_THREADS) {
      const uint4 x = philox4x32_10(make_uint4(t, static_cast<uint32_t>(b), g, 1u), static_cast<uint32_t>(seed),
                                    static_cast<uint32_t>(seed >> 32));
      const uint32_t xw[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = static_cast<int>(4 * g + q - f0);
        if (4 * g + q < f0 || i >= n) continue;
        const bool keep = order_key(srow[i]) >= thr;
        const float w = ((lp_of(i) + bsc) / temp);   // the candidate score below, computed the same way
        srow[i] = (keep && w > -INFINITY) ? w + bm_gumbel(xw[q]) : -INFINITY;
      }
    }
    __syncthreads();
  }
  // ---- this row's top 2k
  float ps = INFINITY;
  int pi = -1;           // the last candidate this thread supplied: the next one must come after it
  float my_s;
  int my_i;
  auto rescan = [&]() {
    my_s = -INFINITY;
    my_i = INT_MAX;
    for (int i = tid; i < n; i += BM_THREADS) {
      float sv;
      if constexpr (SAMPLE) sv = srow[i];
      else sv = score_of(i);
      if ((sv < ps || (sv == ps && i > pi)) && bm_better(sv, i, my_s, my_i)) { my_s = sv; my_i = i; }
    }
  };
  rescan();
  for (int q = 0; q < k2; ++q) {
    float sv = my_s;
    int iv = my_i;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float os = __shfl_xor_sync(0xffffffffu, sv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, iv, o);
      if (bm_better(os, oi, sv, iv)) { sv = os; iv = oi; }
    }
    if (lane == 0) { s_f[warp] = sv; s_i[warp] = iv; }
    __syncthreads();
    if (warp == 0) {
      sv = s_f[lane];
      iv = s_i[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float os = __shfl_xor_sync(0xffffffffu, sv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, iv, o);
        if (bm_better(os, oi, sv, iv)) { sv = os; iv = oi; }
      }
      if (lane == 0) { s_ws = sv; s_wi = iv; }
    }
    __syncthreads();
    const float ws = s_ws;
    const int wi = s_wi;
    if (tid == 0) {
      cand_s[r * 2 * BM_MAX_K + q] = ws;
      if constexpr (SAMPLE) {   // an entry without a key is no draw; a draw carries its warped score, recomputed from
                                // its logit exactly as it was staged
        const bool none = wi == INT_MAX || ws == -INFINITY;
        cand_i[r * 2 * BM_MAX_K + q] = none ? BM_SENTINEL + r * 2 * BM_MAX_K + q : j * n + wi;
        cand_w[r * 2 * BM_MAX_K + q] = none ? -INFINITY : ((lp_of(wi) + bsc) / temp);
      } else {
        cand_i[r * 2 * BM_MAX_K + q] = wi == INT_MAX ? BM_SENTINEL + r * 2 * BM_MAX_K + q : j * n + wi;
      }
    }
    if (wi != INT_MAX && wi % BM_THREADS == tid) { ps = ws; pi = wi; rescan(); }
  }

  // ---- arrival: the last CTA of request b goes on
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(&counters[b], 1) == k - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int r0 = b * k, nc = k * k2;
  if constexpr (SAMPLE) {
    // the request's 2k draws are its top 2k keys; they are then ranked by warped score (ties to the lower flat index)
    __shared__ float m_w[BM_MAX_K * 2 * BM_MAX_K];
    __shared__ float d_w[2 * BM_MAX_K];
    __shared__ int d_i[2 * BM_MAX_K];
    for (int c = tid; c < nc; c += BM_THREADS) {
      const int idx = (r0 + c / k2) * 2 * BM_MAX_K + c % k2;
      m_s[c] = __ldcg(&cand_s[idx]);
      m_i[c] = __ldcg(&cand_i[idx]);
      m_w[c] = __ldcg(&cand_w[idx]);
    }
    __syncthreads();
    if (tid < nc) {
      int rank = 0;
      for (int o = 0; o < nc; ++o) rank += bm_better(m_s[o], m_i[o], m_s[tid], m_i[tid]) ? 1 : 0;
      if (rank < k2) { d_w[rank] = m_w[tid]; d_i[rank] = m_i[tid]; }
    }
    __syncthreads();
    if (tid < k2) {
      int rank = 0;
      for (int o = 0; o < k2; ++o) rank += bm_better(d_w[o], d_i[o], d_w[tid], d_i[tid]) ? 1 : 0;
      t_s[rank] = d_w[tid];
      t_i[rank] = d_i[tid];
    }
  } else {
    for (int c = tid; c < nc; c += BM_THREADS) {
      const int idx = (r0 + c / k2) * 2 * BM_MAX_K + c % k2;
      m_s[c] = __ldcg(&cand_s[idx]);
      m_i[c] = __ldcg(&cand_i[idx]);
    }
    __syncthreads();
    if (tid < nc) {   // rank by counting: flat indices are distinct, so the ranks are a permutation
      int rank = 0;
      for (int o = 0; o < nc; ++o) rank += bm_better(m_s[o], m_i[o], m_s[tid], m_i[tid]) ? 1 : 0;
      if (rank < k2) { t_s[rank] = m_s[tid]; t_i[rank] = m_i[tid]; }
    }
  }
  __syncthreads();

  // ---- the scorer (BeamSearchScorer.process + BeamHypotheses.add / is_done), serial over 2k candidates
  if (tid == 0) {
    const int t = kv_len[r0] - prompt_len[r0];   // tokens generated before this step
    const int pad = prm->pad_token_id, in_len = prm->input_len, es = prm->early_stopping;
    const double lp = prm->length_penalty;
    for (int c = 0; c < k; ++c) h_src[c] = -1;
    if (done[b]) {
      for (int c = 0; c < k; ++c) { c_par[c] = r0 + c; c_tok[c] = pad; c_sc[c] = 0.f; }
    } else {
      int cnt = hyp_count[b], filled = 0;
      auto worst = [&]() -> double {
        double w = 1e9;
        for (int s = 0; s < cnt; ++s) w = fmin(w, hyp_score[r0 + s]);
        return w;
      };
      for (int q = 0; q < k2 && filled < k; ++q) {
        const int f = t_i[q];
        if (f >= BM_SENTINEL) break;
        const int bj = f / n, tok = f % n;
        bool eos = false;
        for (int e = 0; e < prm->n_eos; ++e) eos |= prm->eos[e] == tok;
        if (eos) {
          if (q >= k) continue;
          const int L = in_len + t;
          const double sc = static_cast<double>(t_s[q]) / pow(static_cast<double>(L), lp);
          if (cnt < k || sc > worst()) {
            int slot = cnt;
            if (cnt < k) {
              ++cnt;
            } else {   // evict the lowest score, the earliest added among equals
              slot = 0;
              for (int s = 1; s < cnt; ++s)
                if (hyp_score[r0 + s] < hyp_score[r0 + slot] ||
                    (hyp_score[r0 + s] == hyp_score[r0 + slot] && hyp_seq[r0 + s] < hyp_seq[r0 + slot]))
                  slot = s;
            }
            hyp_score[r0 + slot] = sc;
            hyp_len[r0 + slot] = L;
            hyp_seq[r0 + slot] = t * 2 * BM_MAX_K + q;
            h_src[slot] = r0 + bj;
          }
        } else {
          c_par[filled] = r0 + bj; c_tok[filled] = tok; c_sc[filled] = t_s[q];
          ++filled;
        }
      }
      for (; filled < k; ++filled) { c_par[filled] = r0 + filled; c_tok[filled] = pad; c_sc[filled] = -1e9f; }
      hyp_count[b] = cnt;
      if (cnt >= k) {
        bool d = true;
        if (es != 1) {
          const double len = (es == 2 && lp > 0.0) ? static_cast<double>(prm->max_length) : static_cast<double>(in_len + t);
          d = worst() >= static_cast<double>(t_s[0]) / pow(len, lp);
        }
        if (d) done[b] = 1;
      }
    }
    s_t = t;
    s_P = prompt_len[r0];
  }
  __syncthreads();
  const int t = s_t, P = s_P;

  // ---- generated ids of this step's new hypotheses: token j of row p's history was logged by row beam_src[p][P + j]
  for (int x = tid; x < k * t; x += BM_THREADS) {
    const int slot = x / t, jj = x % t, p = h_src[slot];
    if (p < 0 || jj >= hyp_ld || P + jj >= src_ld || jj >= log_stride) continue;
    const int w = beam_src[static_cast<long long>(p) * src_ld + P + jj];
    hyp_ids[static_cast<long long>(r0 + slot) * hyp_ld + jj] = token_log[static_cast<long long>(w) * log_stride + jj];
  }
  __syncthreads();
  // ---- children take their parent's history; every parent column is read before any child column is written
  const int end = min(P + t, src_ld);
  for (int c0 = P; c0 < end; c0 += BM_STAGE) {
    const int w = min(BM_STAGE, end - c0);
    for (int x = tid; x < k * w; x += BM_THREADS)
      stage[x / w][x % w] = beam_src[static_cast<long long>(c_par[x / w]) * src_ld + c0 + x % w];
    __syncthreads();
    for (int x = tid; x < k * w; x += BM_THREADS)
      beam_src[static_cast<long long>(r0 + x / w) * src_ld + c0 + x % w] = stage[x / w][x % w];
    __syncthreads();
  }
  if (tid < k) {
    const int rr = r0 + tid;
    beam_score[rr] = c_sc[tid];
    parent[rr] = c_par[tid];
    next_src[rr] = c_tok[tid];
    if (t >= 0 && t < log_stride) token_log[static_cast<long long>(rr) * log_stride + t] = c_tok[tid];
    if (P + t < src_ld) beam_src[static_cast<long long>(rr) * src_ld + P + t] = rr;   // the child writes position P + t next
    positions[rr] += 1;
    kv_len[rr] += 1;
  }
  if (tid == 0) counters[b] = 0;
}

// ------------------------------------------------------------------ logits processors (HF 4.31 repetition penalty,
// no-repeat n-grams, min_length, min_new_tokens), in place on rows of fp32 scores. One CTA per row. The row's history
// (its raw prompt ids, then its generated ids, read through beam_src for beam rows) is staged in shared memory; every
// write of a pass goes to a distinct entry or writes the same -inf, and the passes are separated by barriers, so the
// result does not depend on thread order.
constexpr int LP_MAX_N = 49152;
constexpr int LP_MAX_HIST = 8192;   // staged history tokens per row (32 KB)

template <bool LOGPROBS>
__global__ void __launch_bounds__(BM_THREADS, 1)
logits_process_kernel(float* __restrict__ logits, long long ld, int n, const vb_proc_params* __restrict__ prm,
                      const int32_t* __restrict__ prompt_ids, int prompt_ld, const int64_t* __restrict__ token_log,
                      int log_stride, const int32_t* __restrict__ beam_src, int src_ld,
                      const int32_t* __restrict__ kv_len, const int32_t* __restrict__ prompt_len) {
  __shared__ int32_t hist[LP_MAX_HIST];
  __shared__ uint32_t seen[LP_MAX_N / 32];
  __shared__ float s_f[32];
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_wait();      // the logits and the decode state come from the predecessors
  pdl_trigger();
  float* row = logits + r * ld;
  if constexpr (LOGPROBS) {
    // the beam kernel's log-softmax, in its reduction order: (x - max) - log(sum exp(x - max)), NaN as -inf
    float mx = -INFINITY;
    for (int i = tid; i < n; i += BM_THREADS) {
      float v = row[i];
      if (v != v) v = -INFINITY;
      mx = fmaxf(mx, v);
    }
    mx = bm_block_max(mx, s_f, lane, warp);
    float sum = 0.f;
    if (mx > -INFINITY)
      for (int i = tid; i < n; i += BM_THREADS) {
        float v = row[i];
        if (v != v) v = -INFINITY;
        sum += expf(v - mx);
      }
    const float logz = logf(bm_block_sum(sum, s_f, lane, warp));
    for (int i = tid; i < n; i += BM_THREADS) {
      float v = row[i];
      if (v != v) v = -INFINITY;
      row[i] = mx == -INFINITY ? -INFINITY : (v - mx) - logz;
    }
    __syncthreads();
  }
  const float penalty = prm->repetition_penalty;
  const int ngram = prm->no_repeat_ngram_size;
  const bool counted = kv_len != nullptr && prompt_len != nullptr;
  const int t = counted ? min(max(kv_len[r] - prompt_len[r], 0), log_stride) : 0;   // generated tokens so far
  const int P = counted ? prompt_len[r] : 0;
  const int in_len = min(max(prm->input_len, 0), prompt_ld);
  const int L = in_len + t;                       // cur_len = input_ids.shape[-1]; <= LP_MAX_HIST (checked at launch)
  const int words = (n + 31) >> 5;
  if (penalty != 1.f || ngram > 0) {
    for (int j = tid; j < L; j += BM_THREADS) {
      int32_t tok;
      if (j < in_len) {
        tok = prompt_ids[static_cast<long long>(r) * prompt_ld + j];
      } else {
        const int g = j - in_len;
        const int src = (beam_src != nullptr && P + g < src_ld) ? beam_src[static_cast<long long>(r) * src_ld + P + g] : r;
        tok = static_cast<int32_t>(token_log[static_cast<long long>(src) * log_stride + g]);
      }
      hist[j] = tok;
    }
    for (int w = tid; w < words; w += BM_THREADS) seen[w] = 0u;
    __syncthreads();
    if (penalty != 1.f) {
      // mark each in-vocabulary id once (sentinels < 0 are skipped), then penalise every marked entry once
      for (int j = tid; j < L; j += BM_THREADS) {
        const int tok = hist[j];
        if (tok >= 0 && tok < n) atomicOr(&seen[tok >> 5], 1u << (tok & 31));
      }
      __syncthreads();
      for (int w = tid; w < words; w += BM_THREADS) {
        uint32_t bits = seen[w];
        while (bits) {
          const int i = (w << 5) + __ffs(bits) - 1;
          bits &= bits - 1u;
          const float s = row[i];
          row[i] = s < 0.f ? __fmul_rn(s, penalty) : __fdiv_rn(s, penalty);
        }
      }
      __syncthreads();
    }
    if (ngram > 0 && L + 1 >= ngram) {
      // window s (0 <= s <= L - ngram) whose first ngram - 1 tokens equal the last ngram - 1 bans its last token
      const int tail = L - ngram + 1;
      for (int s = tid; s <= L - ngram; s += BM_THREADS) {
        bool match = true;
        for (int q = 0; q < ngram - 1 && match; ++q) match = hist[s + q] == hist[tail + q];
        const int tok = hist[s + ngram - 1];
        if (match && tok >= 0 && tok < n) row[tok] = -INFINITY;
      }
    }
  }
  if (tid == 0 && ((prm->min_length > 0 && L < prm->min_length) || (prm->min_new_tokens > 0 && t < prm->min_new_tokens))) {
    const int n_eos = min(max(prm->n_eos, 0), 8);
    for (int e = 0; e < n_eos; ++e) {
      const int tok = prm->eos[e];
      if (tok >= 0 && tok < n) row[tok] = -INFINITY;
    }
  }
}

}  // namespace vb

using namespace vb;

extern "C" int vb200_argmax_advance(const float* logits, int64_t ld, int64_t rows, int64_t n, int64_t* out_idx,
                                    int32_t* next_src, int32_t* positions, int32_t* kv_len, int64_t* token_log,
                                    int64_t log_stride, const int32_t* prompt_len, cudaStream_t stream) {
  VB_CHECK_ARG(logits && out_idx && rows > 0 && n > 0);
  VB_CHECK_ARG(token_log == nullptr || (kv_len != nullptr && prompt_len != nullptr));
  cudaError_t e = vb_launch(argmax_advance_kernel, dim3(static_cast<unsigned>(rows)), dim3(1024), 0, stream, logits,
                            static_cast<long long>(ld), static_cast<int>(n), out_idx, next_src, positions, kv_len,
                            token_log, static_cast<int>(log_stride), prompt_len);
  if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
  return VB_OK;
}

extern "C" int vb200_sample_advance(const float* logits, int64_t ld, int64_t rows, int64_t n,
                                    const vb_sample_params* params, int64_t* out_idx, int32_t* next_src,
                                    int32_t* positions, int32_t* kv_len, int64_t* token_log, int64_t log_stride,
                                    const int32_t* prompt_len, cudaStream_t stream) {
  VB_CHECK_ARG(logits && params && rows > 0 && rows <= INT_MAX && n > 0 && ld >= n);
  VB_CHECK_ARG(token_log == nullptr ||
               (kv_len != nullptr && prompt_len != nullptr && log_stride > 0 && log_stride <= INT_MAX));
  if (n > SMP_MAX_N) return VB_ERR_UNSUPPORTED;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(sample_advance_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         SMP_MAX_N * static_cast<int>(sizeof(float)));
    if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
    attr_set = true;
  }
  cudaError_t e = vb_launch(sample_advance_kernel, dim3(static_cast<unsigned>(rows)), dim3(SMP_THREADS),
                            static_cast<size_t>(n) * sizeof(float), stream, logits, static_cast<long long>(ld),
                            static_cast<int>(n), params, out_idx, next_src, positions, kv_len, token_log,
                            static_cast<int>(log_stride), prompt_len);
  if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
  return VB_OK;
}

extern "C" size_t vb200_beam_workspace_size(int64_t rows) {
  // [counters | candidate scores | flat indices | warped scores (beam sampling)] x 2 * BM_MAX_K per row
  return BM_COUNTER_BYTES + static_cast<size_t>(rows > 0 ? rows : 0) * 2 * BM_MAX_K * (2 * sizeof(float) + sizeof(int32_t));
}

template <bool SAMPLE, bool LOGPROBS = false>
static int launch_beam_advance(const float* logits, int64_t ld, int64_t B, int64_t k, int64_t n,
                               const vb_beam_params* params, float* beam_score, int32_t* parent, int32_t* done,
                               int32_t* beam_src, int64_t src_ld, double* hyp_score, int32_t* hyp_len, int32_t* hyp_seq,
                               int32_t* hyp_count, int64_t* hyp_ids, int64_t hyp_ld, int32_t* next_src, int32_t* positions,
                               int32_t* kv_len, int64_t* token_log, int64_t log_stride, const int32_t* prompt_len,
                               void* workspace, size_t workspace_bytes, const vb_sample_params* sample_params,
                               cudaStream_t stream) {
  VB_CHECK_ARG(logits && params && beam_score && parent && done && beam_src && hyp_score && hyp_len && hyp_seq &&
               hyp_count && hyp_ids && next_src && positions && kv_len && token_log && prompt_len);
  VB_CHECK_ARG(B > 0 && k > 0 && n >= 2 && ld >= n && src_ld > 0 && src_ld <= INT_MAX && hyp_ld > 0 &&
               hyp_ld <= INT_MAX && log_stride > 0 && log_stride <= INT_MAX);
  if (k > BM_MAX_K || n > BM_MAX_N || B > static_cast<int64_t>(BM_COUNTER_BYTES / sizeof(int32_t)))
    return VB_ERR_UNSUPPORTED;
  const int64_t rows = B * k;
  if (!workspace || workspace_bytes < vb200_beam_workspace_size(rows)) return VB_ERR_WORKSPACE;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(beam_advance_kernel<SAMPLE, LOGPROBS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         BM_MAX_N * static_cast<int>(sizeof(float)));
    if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
    attr_set = true;
  }
  int32_t* counters = reinterpret_cast<int32_t*>(workspace);
  float* cand_s = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + BM_COUNTER_BYTES);
  int32_t* cand_i = reinterpret_cast<int32_t*>(cand_s + rows * 2 * BM_MAX_K);
  float* cand_w = reinterpret_cast<float*>(cand_i + rows * 2 * BM_MAX_K);
  cudaError_t e = vb_launch(beam_advance_kernel<SAMPLE, LOGPROBS>, dim3(static_cast<unsigned>(rows)), dim3(BM_THREADS),
                            static_cast<size_t>(n) * sizeof(float), stream, logits, static_cast<long long>(ld),
                            static_cast<int>(n), static_cast<int>(k), params, beam_score, parent, done, beam_src,
                            static_cast<int>(src_ld), hyp_score, hyp_len, hyp_seq, hyp_count, hyp_ids,
                            static_cast<int>(hyp_ld), next_src, positions, kv_len, token_log,
                            static_cast<int>(log_stride), prompt_len, cand_s, cand_i, counters, sample_params, cand_w);
  if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
  return VB_OK;
}

extern "C" int vb200_beam_advance(const float* logits, int64_t ld, int64_t B, int64_t k, int64_t n,
                                  const vb_beam_params* params, float* beam_score, int32_t* parent, int32_t* done,
                                  int32_t* beam_src, int64_t src_ld, double* hyp_score, int32_t* hyp_len,
                                  int32_t* hyp_seq, int32_t* hyp_count, int64_t* hyp_ids, int64_t hyp_ld,
                                  int32_t* next_src, int32_t* positions, int32_t* kv_len, int64_t* token_log,
                                  int64_t log_stride, const int32_t* prompt_len, void* workspace,
                                  size_t workspace_bytes, cudaStream_t stream) {
  return launch_beam_advance<false>(logits, ld, B, k, n, params, beam_score, parent, done, beam_src, src_ld, hyp_score,
                                    hyp_len, hyp_seq, hyp_count, hyp_ids, hyp_ld, next_src, positions, kv_len,
                                    token_log, log_stride, prompt_len, workspace, workspace_bytes, nullptr, stream);
}

extern "C" int vb200_beam_sample_advance(const float* logits, int64_t ld, int64_t B, int64_t k, int64_t n,
                                         const vb_beam_params* params, float* beam_score, int32_t* parent,
                                         int32_t* done, int32_t* beam_src, int64_t src_ld, double* hyp_score,
                                         int32_t* hyp_len, int32_t* hyp_seq, int32_t* hyp_count, int64_t* hyp_ids,
                                         int64_t hyp_ld, int32_t* next_src, int32_t* positions, int32_t* kv_len,
                                         int64_t* token_log, int64_t log_stride, const int32_t* prompt_len,
                                         void* workspace, size_t workspace_bytes, const vb_sample_params* sample_params,
                                         cudaStream_t stream) {
  VB_CHECK_ARG(sample_params != nullptr);
  return launch_beam_advance<true>(logits, ld, B, k, n, params, beam_score, parent, done, beam_src, src_ld, hyp_score,
                                   hyp_len, hyp_seq, hyp_count, hyp_ids, hyp_ld, next_src, positions, kv_len, token_log,
                                   log_stride, prompt_len, workspace, workspace_bytes, sample_params, stream);
}

extern "C" int vb200_beam_advance_logprobs(const float* logits, int64_t ld, int64_t B, int64_t k, int64_t n,
                                           const vb_beam_params* params, float* beam_score, int32_t* parent,
                                           int32_t* done, int32_t* beam_src, int64_t src_ld, double* hyp_score,
                                           int32_t* hyp_len, int32_t* hyp_seq, int32_t* hyp_count, int64_t* hyp_ids,
                                           int64_t hyp_ld, int32_t* next_src, int32_t* positions, int32_t* kv_len,
                                           int64_t* token_log, int64_t log_stride, const int32_t* prompt_len,
                                           void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return launch_beam_advance<false, true>(logits, ld, B, k, n, params, beam_score, parent, done, beam_src, src_ld,
                                          hyp_score, hyp_len, hyp_seq, hyp_count, hyp_ids, hyp_ld, next_src, positions,
                                          kv_len, token_log, log_stride, prompt_len, workspace, workspace_bytes, nullptr,
                                          stream);
}

extern "C" int vb200_beam_sample_advance_logprobs(const float* logits, int64_t ld, int64_t B, int64_t k, int64_t n,
                                                  const vb_beam_params* params, float* beam_score, int32_t* parent,
                                                  int32_t* done, int32_t* beam_src, int64_t src_ld, double* hyp_score,
                                                  int32_t* hyp_len, int32_t* hyp_seq, int32_t* hyp_count,
                                                  int64_t* hyp_ids, int64_t hyp_ld, int32_t* next_src,
                                                  int32_t* positions, int32_t* kv_len, int64_t* token_log,
                                                  int64_t log_stride, const int32_t* prompt_len, void* workspace,
                                                  size_t workspace_bytes, const vb_sample_params* sample_params,
                                                  cudaStream_t stream) {
  VB_CHECK_ARG(sample_params != nullptr);
  return launch_beam_advance<true, true>(logits, ld, B, k, n, params, beam_score, parent, done, beam_src, src_ld,
                                         hyp_score, hyp_len, hyp_seq, hyp_count, hyp_ids, hyp_ld, next_src, positions,
                                         kv_len, token_log, log_stride, prompt_len, workspace, workspace_bytes,
                                         sample_params, stream);
}

extern "C" int vb200_logits_process(float* logits, int64_t ld, int64_t rows, int64_t n, const vb_proc_params* params,
                                    const int32_t* prompt_ids, int64_t prompt_ld, const int64_t* token_log,
                                    int64_t log_stride, const int32_t* beam_src, int64_t src_ld, const int32_t* kv_len,
                                    const int32_t* prompt_len, int logprobs, cudaStream_t stream) {
  VB_CHECK_ARG(logits && params && prompt_ids && rows > 0 && rows <= INT_MAX && n > 0 && ld >= n && prompt_ld > 0 &&
               prompt_ld <= INT_MAX);
  VB_CHECK_ARG((kv_len == nullptr) == (prompt_len == nullptr));
  VB_CHECK_ARG(kv_len == nullptr || (token_log != nullptr && log_stride > 0 && log_stride <= INT_MAX));
  VB_CHECK_ARG(beam_src == nullptr || (kv_len != nullptr && src_ld > 0 && src_ld <= INT_MAX));
  if (n > LP_MAX_N || prompt_ld + (kv_len != nullptr ? log_stride : 0) > LP_MAX_HIST) return VB_ERR_UNSUPPORTED;
  const int ls = kv_len != nullptr ? static_cast<int>(log_stride) : 0;
  const int sl = beam_src != nullptr ? static_cast<int>(src_ld) : 0;
  cudaError_t e = logprobs
      ? vb_launch(logits_process_kernel<true>, dim3(static_cast<unsigned>(rows)), dim3(BM_THREADS), 0, stream, logits,
                  static_cast<long long>(ld), static_cast<int>(n), params, prompt_ids, static_cast<int>(prompt_ld),
                  token_log, ls, beam_src, sl, kv_len, prompt_len)
      : vb_launch(logits_process_kernel<false>, dim3(static_cast<unsigned>(rows)), dim3(BM_THREADS), 0, stream, logits,
                  static_cast<long long>(ld), static_cast<int>(n), params, prompt_ids, static_cast<int>(prompt_ld),
                  token_log, ls, beam_src, sl, kv_len, prompt_len);
  if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
  return VB_OK;
}

extern "C" int vb200_rope_kv_append(void* qkv, int64_t ld_qkv, const int32_t* positions,
                                    const int32_t* batch_of_token, const int32_t* slot_of_token,
                                    void* k_pages, void* v_pages, const int32_t* block_table,
                                    int64_t max_pages, int64_t tokens, int64_t n_heads,
                                    int64_t head_dim, int64_t page_size, float rope_theta,
                                    cudaStream_t stream) {
  VB_CHECK_ARG(qkv && positions && tokens >= 0 && n_heads > 0);
  VB_CHECK_ARG(head_dim % 16 == 0 && ld_qkv % 8 == 0 && ld_qkv >= 3 * n_heads * head_dim);
  VB_CHECK_ARG((k_pages == nullptr) == (v_pages == nullptr));
  VB_CHECK_ARG(k_pages == nullptr || (block_table != nullptr && page_size > 0 && max_pages > 0));
  if (tokens == 0) return VB_OK;
  rope_kv_append_kernel<<<static_cast<unsigned>(tokens), 256, 0, stream>>>(
      reinterpret_cast<bf16*>(qkv), ld_qkv, positions, batch_of_token, slot_of_token,
      reinterpret_cast<bf16*>(k_pages), reinterpret_cast<bf16*>(v_pages), block_table,
      static_cast<int>(max_pages), static_cast<int>(n_heads), static_cast<int>(head_dim),
      static_cast<int>(page_size), log2f(rope_theta));
  VB_LAUNCH_CHECK();
  return VB_OK;
}

static int decode_splits(int64_t max_kv_len, int64_t bh) {
  // As few splits as still give every SM its 4 resident CTAs (113 registers x 128 threads): the whole grid runs as ONE
  // wave and the per-CTA fixed cost (q load + RoPE, partial write, arrival atomics, merge) is paid once per 512 keys, with
  // the first two pages already on their way to L2 before the dependency wait. Small batches get more, shorter splits (down
  // to 128 keys) to fill the machine.
  static int keys_env = -1;   // VB200_DEC_SPLIT_KEYS = 128 / 256 / 512 pins the split length (tuning aid)
  if (keys_env < 0) {
    const char* e = getenv("VB200_DEC_SPLIT_KEYS");
    const int v = e ? atoi(e) : 0;
    keys_env = (v == 128 || v == 256 || v == 512) ? v : 0;
  }
  int s;
  if (keys_env) {
    s = static_cast<int>((max_kv_len + keys_env - 1) / keys_env);
  } else {
    const int s_min = static_cast<int>((max_kv_len + DEC_CHUNK - 1) / DEC_CHUNK);          // a split is at most 512 keys
    const int s_max = static_cast<int>((max_kv_len + 127) / 128);                           // ... and at least 128
    int s_fill = static_cast<int>(4LL * vb_num_sms() / (bh > 0 ? bh : 1));                  // one wave of 4 CTAs per SM
    if (s_fill > s_max) s_fill = s_max;
    s = s_fill > s_min ? s_fill : s_min;
  }
  if (s < 1) s = 1;
  if (s > 32) s = 32;
  return s;
}

// The arrival counters live in a FIXED-size prefix: the partial regions behind it move with (B, n_heads, splits), and a
// workspace that serves calls of different batch sizes (one CUDA graph per batch size replays against the same buffer) must
// never see a later call's counters where an earlier call left partial results (stale non-zero "counters" = a merge that
// fires early or never).
constexpr size_t DEC_COUNTER_BYTES = 16384;   // B * n_heads <= 4096

extern "C" size_t vb200_attn_decode_workspace_size(int64_t B, int64_t n_heads, int64_t head_dim,
                                                   int64_t max_splits) {
  // [arrival counters: 16 KB | (m, l) per split | unnormalised o per split]; zero-fill ONCE before first use
  if (max_splits < 1) max_splits = 32;
  return DEC_COUNTER_BYTES + static_cast<size_t>(B) * n_heads * max_splits * (head_dim + 2) * sizeof(float);
}

static int launch_attn_decode(const void* q, int64_t ld_q, void* k_pages, void* v_pages,
                              const int32_t* block_table, int64_t max_pages, const int32_t* kv_len, void* out,
                              int64_t ld_o, int64_t B, int64_t n_heads, int64_t head_dim, int64_t page_size,
                              int64_t max_kv_len, float scale, void* workspace, size_t workspace_bytes,
                              const float* rope_table, cudaStream_t stream, const int32_t* beam_src = nullptr,
                              int64_t src_ld = 0, const int32_t* gen_start = nullptr) {
  VB_CHECK_ARG(q && k_pages && v_pages && block_table && kv_len && out);
  VB_CHECK_ARG(B > 0 && n_heads > 0 && page_size > 0 && max_pages > 0);
  if (head_dim != 128) return VB_ERR_UNSUPPORTED;
  VB_CHECK_ARG(ld_q % 8 == 0);
  if (page_size != 64) return VB_ERR_UNSUPPORTED;  // one 64-key trip == one page
  const int splits = decode_splits(max_kv_len, B * n_heads);
  int per = static_cast<int>((max_kv_len + splits - 1) / splits);
  per = (per + 63) / 64 * 64;
  if (per > DEC_CHUNK) return VB_ERR_ARG;
  float* ws_ml = nullptr;
  float* ws_o = nullptr;
  int* counters = nullptr;
  if (splits > 1) {
    size_t need = vb200_attn_decode_workspace_size(B, n_heads, head_dim, splits);
    if (!workspace || workspace_bytes < need) return VB_ERR_WORKSPACE;
    if (static_cast<size_t>(B) * n_heads * sizeof(int) > DEC_COUNTER_BYTES) return VB_ERR_UNSUPPORTED;
    counters = reinterpret_cast<int*>(workspace);
    ws_ml = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + DEC_COUNTER_BYTES);
    ws_o = ws_ml + static_cast<size_t>(B) * n_heads * splits * 2;
  }
  dim3 grid(splits, static_cast<unsigned>(n_heads), static_cast<unsigned>(B));
  cudaError_t e;
#define VB_LAUNCH_DECODE(ROPE_, TRIPS_, TABLE_, ...)                                                               \
  e = vb_launch(attn_decode_kernel<ROPE_, TRIPS_, ##__VA_ARGS__>, grid, dim3(DEC_THREADS), 0, stream,             \
                reinterpret_cast<const bf16*>(q), static_cast<long long>(ld_q), reinterpret_cast<bf16*>(k_pages), \
                reinterpret_cast<bf16*>(v_pages), block_table, static_cast<int>(max_pages), kv_len,                \
                static_cast<int>(n_heads), static_cast<int>(page_size), scale, splits, per, ws_ml, ws_o, counters, \
                reinterpret_cast<bf16*>(out), static_cast<long long>(ld_o), TABLE_, beam_src,                      \
                static_cast<int>(src_ld), gen_start)
  const float* no_table = nullptr;
  if (beam_src != nullptr) {
    if (per <= DEC_CHUNK / 2) VB_LAUNCH_DECODE(true, DEC_CHUNK / 128, rope_table, true);
    else VB_LAUNCH_DECODE(true, DEC_CHUNK / 64, rope_table, true);
  } else if (rope_table != nullptr) {
    if (per <= DEC_CHUNK / 2) VB_LAUNCH_DECODE(true, DEC_CHUNK / 128, rope_table);
    else VB_LAUNCH_DECODE(true, DEC_CHUNK / 64, rope_table);
  } else {
    if (per <= DEC_CHUNK / 2) VB_LAUNCH_DECODE(false, DEC_CHUNK / 128, no_table);
    else VB_LAUNCH_DECODE(false, DEC_CHUNK / 64, no_table);
  }
#undef VB_LAUNCH_DECODE
  if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
  return VB_OK;
}

extern "C" int vb200_attn_decode_paged(const void* q, int64_t ld_q, const void* k_pages,
                                       const void* v_pages, const int32_t* block_table,
                                       int64_t max_pages, const int32_t* kv_len, void* out,
                                       int64_t ld_o, int64_t B, int64_t n_heads, int64_t head_dim,
                                       int64_t page_size, int64_t max_kv_len, float scale,
                                       void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return launch_attn_decode(q, ld_q, const_cast<void*>(k_pages), const_cast<void*>(v_pages), block_table, max_pages,
                            kv_len, out, ld_o, B, n_heads, head_dim, page_size, max_kv_len, scale, workspace,
                            workspace_bytes, nullptr, stream);
}

extern "C" int vb200_rope_table(const int32_t* positions, float* table, int64_t B, int64_t head_dim, float rope_theta,
                                cudaStream_t stream) {
  VB_CHECK_ARG(positions && table && B > 0 && head_dim > 0 && head_dim % 2 == 0 && head_dim <= 2048);
  cudaError_t e = vb_launch(rope_table_kernel, dim3(static_cast<unsigned>(B)),
                            dim3(static_cast<unsigned>((head_dim / 2 + 31) / 32 * 32)), 0, stream, positions, table,
                            static_cast<int>(head_dim / 2), log2f(rope_theta));
  if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
  return VB_OK;
}

extern "C" int vb200_attn_decode_rope(const void* qkv, int64_t ld_qkv, const float* rope_table, void* k_pages,
                                      void* v_pages, const int32_t* block_table, int64_t max_pages,
                                      const int32_t* kv_len, void* out, int64_t ld_o, int64_t B,
                                      int64_t n_heads, int64_t head_dim, int64_t page_size,
                                      int64_t max_kv_len, float scale, void* workspace,
                                      size_t workspace_bytes, cudaStream_t stream) {
  VB_CHECK_ARG(rope_table != nullptr && ld_qkv >= 3 * n_heads * head_dim);
  return launch_attn_decode(qkv, ld_qkv, k_pages, v_pages, block_table, max_pages, kv_len, out, ld_o, B, n_heads,
                            head_dim, page_size, max_kv_len, scale, workspace, workspace_bytes, rope_table, stream);
}

extern "C" int vb200_attn_decode_rope_beam(const void* qkv, int64_t ld_qkv, const float* rope_table, void* k_pages,
                                           void* v_pages, const int32_t* block_table, int64_t max_pages,
                                           const int32_t* kv_len, const int32_t* beam_src, int64_t src_ld,
                                           const int32_t* gen_start, void* out, int64_t ld_o, int64_t B,
                                           int64_t n_heads, int64_t head_dim, int64_t page_size, int64_t max_kv_len,
                                           float scale, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  VB_CHECK_ARG(rope_table != nullptr && ld_qkv >= 3 * n_heads * head_dim);
  VB_CHECK_ARG(beam_src != nullptr && gen_start != nullptr && src_ld >= max_kv_len && src_ld <= INT_MAX);
  return launch_attn_decode(qkv, ld_qkv, k_pages, v_pages, block_table, max_pages, kv_len, out, ld_o, B, n_heads,
                            head_dim, page_size, max_kv_len, scale, workspace, workspace_bytes, rope_table, stream,
                            beam_src, src_ld, gen_start);
}

extern "C" int vb200_splice_multimodal(const void* embed, int64_t vocab, const void* feats,
                                       int64_t n_feat_rows, const int32_t* srcmap, void* out,
                                       int64_t rows, int64_t d, cudaStream_t stream) {
  VB_CHECK_ARG(embed && srcmap && out && d > 0 && d % 8 == 0 && rows >= 0);
  VB_CHECK_ARG(feats != nullptr || n_feat_rows == 0);
  if (rows == 0) return VB_OK;
  cudaError_t e = vb_launch(splice_kernel, dim3(static_cast<unsigned>(rows)), dim3(256), 0, stream,
                            reinterpret_cast<const bf16*>(embed), static_cast<long long>(vocab),
                            reinterpret_cast<const bf16*>(feats), static_cast<long long>(n_feat_rows), srcmap,
                            reinterpret_cast<bf16*>(out), static_cast<int>(d));
  if (e != cudaSuccess) { vb_set_last_error(e); return VB_ERR_CUDA; }
  return VB_OK;
}

extern "C" int vb200_argmax_rows(const void* logits, int is_fp32, int64_t ld, int64_t rows, int64_t n,
                                 int64_t* out_idx, cudaStream_t stream) {
  VB_CHECK_ARG(logits && out_idx && rows >= 0 && n > 0);
  if (rows == 0) return VB_OK;
  if (is_fp32)
    argmax_kernel<float><<<static_cast<unsigned>(rows), 1024, 0, stream>>>(reinterpret_cast<const float*>(logits), ld, static_cast<int>(n), out_idx);
  else
    argmax_kernel<bf16><<<static_cast<unsigned>(rows), 1024, 0, stream>>>(reinterpret_cast<const bf16*>(logits), ld, static_cast<int>(n), out_idx);
  VB_LAUNCH_CHECK();
  return VB_OK;
}
