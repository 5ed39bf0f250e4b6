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

template <bool ROPE, int MAX_TRIPS>
__global__ void __launch_bounds__(DEC_THREADS, 4)   // 4 CTAs per SM: the one-wave split policy counts on 4 x (SM count) slots
attn_decode_kernel(const bf16* __restrict__ q, long long ld_q, bf16* __restrict__ k_pages,
                   bf16* __restrict__ v_pages, const int32_t* __restrict__ block_table, int max_pages,
                   const int32_t* __restrict__ kv_len, int H, int page_size, float scale, int splits, int per,
                   float* __restrict__ ws_ml, float* __restrict__ ws_o, int* __restrict__ counters,
                   bf16* __restrict__ out, long long ld_o, const float* __restrict__ rope_table) {
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
  // L2 prefetch of this CTA's first page (K and V, 16 KB each for this head) while the predecessor (the qkv projection,
  // which does not touch the cache) drains: pages of earlier tokens are constant during the step. One 128-byte line per
  // 4 lanes; the remaining trips are prefetched two trips ahead inside the loop.
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
      const long long off = pbase + static_cast<long long>(has ? kk : 0) * HD;
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
    if ((hs >> 1) + 2 < MAX_TRIPS && c0 + 64 * ((hs >> 1) + 2) < c1) prefetch_page(pg[(hs >> 1) + 2]);   // two pages ahead -> L2
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
  // the next page already on its way to L2 while a 64-key trip is processed. Small batches get more, shorter splits (down
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
                              const float* rope_table, cudaStream_t stream) {
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
#define VB_LAUNCH_DECODE(ROPE_, TRIPS_, TABLE_)                                                                    \
  e = vb_launch(attn_decode_kernel<ROPE_, TRIPS_>, grid, dim3(DEC_THREADS), 0, stream,                            \
                reinterpret_cast<const bf16*>(q), static_cast<long long>(ld_q), reinterpret_cast<bf16*>(k_pages), \
                reinterpret_cast<bf16*>(v_pages), block_table, static_cast<int>(max_pages), kv_len,                \
                static_cast<int>(n_heads), static_cast<int>(page_size), scale, splits, per, ws_ml, ws_o, counters, \
                reinterpret_cast<bf16*>(out), static_cast<long long>(ld_o), TABLE_)
  const float* no_table = nullptr;
  if (rope_table != nullptr) {
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
