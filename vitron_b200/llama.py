"""Vicuna-7B / LLaMA decoder stack on the vitron_b200 kernels.

Replaces the arithmetic of HF transformers 4.31 `LlamaModel` / `LlamaForCausalLM.forward` as
called by the reference at vitron/model/language_model/llava_llama.py:91-102 (the q/k/v/RoPE/KV
sequence is restated in-tree at vitron/train/llama_flash_attn_monkey_patch.py:30-66):

    embed -> 32 x [RMSNorm, QKV, RoPE, causal attention over the KV cache, O, +res,
                   RMSNorm, down(SiLU(gate) * up), +res] -> RMSNorm -> lm_head

Differences in mechanism (not in math): q/k/v and gate/up are single fused GEMMs (weights packed
at load), the KV cache is paged in HBM instead of grown with torch.cat, residual adds / SiLU*mul
live in GEMM epilogues, and the decode step is one CUDA graph with the arg-max (or the sampler) on device.
State-dict names are the reference's (SURVEY.md Appendix B).
"""
from dataclasses import dataclass

import torch

from . import nf4 as _nf4
from . import beam as _beam
from . import ops, processors, sampling

BF16 = torch.bfloat16


@dataclass
class LlamaConfig:
    hidden_size: int = 4096
    intermediate_size: int = 11008
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    vocab_size: int = 32000
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    max_position_embeddings: int = 4096

    @property
    def head_dim(self):
        return self.hidden_size // self.num_attention_heads

    @staticmethod
    def from_any(cfg):
        """Accept an HF LlamaConfig-like object or dict."""
        if isinstance(cfg, LlamaConfig):
            return cfg
        get = (lambda k, d: cfg.get(k, d)) if isinstance(cfg, dict) else (lambda k, d: getattr(cfg, k, d))
        theta = get("rope_theta", None)
        if theta is None:
            rp = get("rope_parameters", None) or {}
            theta = rp.get("rope_theta", 10000.0) if isinstance(rp, dict) else 10000.0
        return LlamaConfig(get("hidden_size", 4096), get("intermediate_size", 11008), get("num_hidden_layers", 32),
                           get("num_attention_heads", 32), get("vocab_size", 32000), get("rms_norm_eps", 1e-5),
                           float(theta), get("max_position_embeddings", 4096))


class PagedKVCache:
    """[layers, 2, num_pages, heads, page_size, head_dim] bf16 + a per-slot block table.

    Pages are handed out from a free list; a sequence slot owns ceil(len / page_size) pages. fork() lets slots share the
    full pages of a prompt: every page carries a reference count and returns to the free list when the last slot holding
    it releases it."""

    def __init__(self, cfg, max_batch, max_seq_len, device, page_size=64):
        self.page_size = page_size
        self.max_pages = (max_seq_len + page_size - 1) // page_size
        self.num_pages = max_batch * self.max_pages
        self.max_batch = max_batch
        self.max_seq_len = self.max_pages * page_size
        L, H, D = cfg.num_hidden_layers, cfg.num_attention_heads, cfg.head_dim
        self.pages = torch.zeros((L, 2, self.num_pages, H, page_size, D), dtype=BF16, device=device)
        self.block_table = torch.zeros((max_batch, self.max_pages), dtype=torch.int32, device=device)
        self._free = list(range(self.num_pages - 1, -1, -1))
        self._owned = [[] for _ in range(max_batch)]
        self._refs = [0] * self.num_pages
        self.device = device

    def reserve(self, slot, length):
        need = (length + self.page_size - 1) // self.page_size
        owned = self._owned[slot]
        if need > self.max_pages:
            raise ValueError(f"sequence of {length} tokens exceeds the cache capacity {self.max_seq_len}")
        changed = False
        while len(owned) < need:
            if not self._free:
                raise RuntimeError("KV cache out of pages")
            owned.append(self._free.pop())
            self._refs[owned[-1]] = 1
            changed = True
        return changed

    def release(self, slot):
        for p in reversed(self._owned[slot]):
            self._refs[p] -= 1
            if self._refs[p] == 0:
                self._free.append(p)
        self._owned[slot] = []

    def fork(self, lens, k):
        """Slots 0..len(lens)-1 hold prompts of lens[b] tokens. Afterwards slot b * k + j (j < k) holds prompt b: its
        full pages are shared, and the partial last page is copied per slot (its valid tokens, every layer), because
        the beams write their first generated tokens into it. Call sync_table() afterwards."""
        B, ps = len(lens), self.page_size
        src = [self._owned[b][:(lens[b] + ps - 1) // ps] for b in range(B)]
        for b in range(B):
            for p in src[b]:
                self._refs[p] += 1                 # held by the fork until the copies are made
        for slot in range(max(B, B * k)):
            self.release(slot)
        copies = []
        for b in range(B):
            full, part = lens[b] // ps, lens[b] % ps
            for j in range(k):
                owned = list(src[b][:full])
                for p in owned:
                    self._refs[p] += 1
                if part:
                    if not self._free:
                        raise RuntimeError("KV cache out of pages")
                    owned.append(self._free.pop())
                    self._refs[owned[-1]] = 1
                    copies.append((src[b][full], owned[-1], part))
                self._owned[b * k + j] = owned
        for old, new, n in copies:
            self.pages[:, :, new, :, :n] = self.pages[:, :, old, :, :n]
        for b in range(B):
            for p in src[b]:
                self._refs[p] -= 1
                if self._refs[p] == 0:
                    self._free.append(p)

    def sync_table(self):
        host = torch.zeros((self.max_batch, self.max_pages), dtype=torch.int32)
        for s, owned in enumerate(self._owned):
            if owned:
                host[s, :len(owned)] = torch.tensor(owned, dtype=torch.int32)
        self.block_table.copy_(host, non_blocking=True)

    def k(self, layer):
        return self.pages[layer, 0]

    def v(self, layer):
        return self.pages[layer, 1]


class LlamaEngine:
    def __init__(self, config, device, max_batch=8, max_seq_len=1024, page_size=64):
        self.cfg = LlamaConfig.from_any(config)
        self.device = torch.device(device)
        self.max_batch = max_batch
        self.cache = PagedKVCache(self.cfg, max_batch, max_seq_len, self.device, page_size)
        self.layers = []
        self.embed = None
        self.lm_head = None
        c = self.cfg
        B = max_batch
        dev = self.device
        # static decode state (addresses are baked into the CUDA graph)
        self.d_src = torch.zeros((B,), dtype=torch.int32, device=dev)
        self.d_pos = torch.zeros((B,), dtype=torch.int32, device=dev)
        self.d_len = torch.zeros((B,), dtype=torch.int32, device=dev)
        self.d_prompt = torch.zeros((B,), dtype=torch.int32, device=dev)
        self.d_bot = torch.arange(B, dtype=torch.int32, device=dev)
        self.d_next = torch.zeros((B,), dtype=torch.int64, device=dev)
        self.d_logits = torch.zeros((B, c.vocab_size), dtype=torch.float32, device=dev)
        self.d_rope = torch.zeros((B, c.head_dim), dtype=torch.float32, device=dev)
        # generated ids land here (column = tokens generated so far); persistent so the decode
        # graph survives across generate() calls
        self.token_log = torch.zeros((B, self.cache.max_seq_len), dtype=torch.int64, device=dev)
        # vb_sample_params read by the sampled step: one captured graph serves every temperature / top-k / top-p / seed
        self.d_sample = torch.zeros((ops.SAMPLE_PARAMS.size,), dtype=torch.uint8, device=dev)
        # logits processors (set_processors): vb_proc_params and every row's raw prompt ids, read by the step's
        # logits_process kernel; proc_on selects the graphs that run it
        self.d_proc = torch.zeros((processors.PARAMS.size,), dtype=torch.uint8, device=dev)
        self.d_proc_prompt = torch.zeros((B, self.cache.max_seq_len), dtype=torch.int32, device=dev)
        self.proc_on = False
        self.beam = None       # beam-search state (start_beam), allocated on first use
        self.beam_k = 0        # beams per request of the current beam search; 0 = no beam search started
        self._graphs = {}
        self.launches_per_step = 0
        self.use_pdl = True
        # the split-KV workspace address is baked into the decode graphs: size it for max_batch once, so a later
        # generate() at a larger batch can never move it under a captured graph
        if self.device.type == "cuda":
            ops.reserve_decode_workspace(max_batch, c.num_attention_heads, c.head_dim, self.device)

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, sd, prefix="", nf4=False):
        """HF names: model.embed_tokens.weight, model.layers.N.self_attn.{q,k,v,o}_proj.weight,
        model.layers.N.mlp.{gate,up,down}_proj.weight, model.layers.N.{input,post_attention}_layernorm.weight,
        model.norm.weight, lm_head.weight.

        nf4=True is the reference's load_4bit (builder.py:36-46): the seven projections of every layer are quantised to NF4
        (vitron_b200.nf4) from the checkpoint tensors, one tensor at a time on the load device; the RMSNorm gains cannot be
        folded into quantised weights and are applied as the kernels' column scale instead. embed_tokens and lm_head stay
        bf16, as bitsandbytes leaves them."""
        if nf4:
            return self._load_nf4(sd, prefix)
        dev = self.device

        def get(name):
            return sd[prefix + name].detach().to(device=dev, dtype=BF16)

        def folded(name, ln):
            # RMSNorm gain folded into the consuming projection: (x * rstd * g) W^T == rstd * x (W diag(g))^T
            w = sd[prefix + name].detach().to(device=dev, dtype=torch.float32)
            return (w * sd[prefix + ln].detach().to(device=dev, dtype=torch.float32)[None, :]).to(BF16)

        self.embed = get("model.embed_tokens.weight").contiguous()
        self.lm_head = folded("lm_head.weight", "model.norm.weight").contiguous()
        self.layers = []
        # the RMSNorm gains are folded into the consuming weights; the (tiny) gain vectors are kept so that state_dict()
        # can hand back reference-named tensors
        g32 = lambda n: sd[prefix + n].detach().to(device=dev, dtype=torch.float32).contiguous()
        self.norm_gains = dict(norm=g32("model.norm.weight"), ln1=[], ln2=[])
        for i in range(self.cfg.num_hidden_layers):
            p = f"model.layers.{i}."
            ln1, ln2 = p + "input_layernorm.weight", p + "post_attention_layernorm.weight"
            self.norm_gains["ln1"].append(g32(ln1))
            self.norm_gains["ln2"].append(g32(ln2))
            wqkv = torch.cat([folded(p + "self_attn.q_proj.weight", ln1), folded(p + "self_attn.k_proj.weight", ln1),
                              folded(p + "self_attn.v_proj.weight", ln1)], 0).contiguous()
            wgu = ops.pack_glu_weight(folded(p + "mlp.gate_proj.weight", ln2), folded(p + "mlp.up_proj.weight", ln2))
            self.layers.append(dict(wqkv=wqkv, wo=get(p + "self_attn.o_proj.weight").contiguous(), wgu=wgu,
                                    wdown=get(p + "mlp.down_proj.weight").contiguous()))
        self._graphs = {}
        return self

    def _load_nf4(self, sd, prefix):
        dev = self.device
        t = lambda n: sd[prefix + n].detach().to(device=dev)
        g32 = lambda n: t(n).to(torch.float32).contiguous()
        q = lambda n: _nf4.quantize(t(n))
        self.embed = t("model.embed_tokens.weight").to(BF16).contiguous()
        gn = g32("model.norm.weight")
        self.lm_head = (t("lm_head.weight").to(torch.float32) * gn[None, :]).to(BF16).contiguous()
        self.norm_gains = dict(norm=gn, ln1=[], ln2=[])
        self.layers = []
        for i in range(self.cfg.num_hidden_layers):
            p = f"model.layers.{i}."
            g1, g2 = g32(p + "input_layernorm.weight"), g32(p + "post_attention_layernorm.weight")
            self.norm_gains["ln1"].append(g1)
            self.norm_gains["ln2"].append(g2)
            wqkv = _nf4.NF4Weight.cat([q(p + "self_attn.q_proj.weight"), q(p + "self_attn.k_proj.weight"),
                                       q(p + "self_attn.v_proj.weight")])
            self.layers.append(dict(wqkv=wqkv, wo=q(p + "self_attn.o_proj.weight"),
                                    wgu=_pack_glu_nf4(q(p + "mlp.gate_proj.weight"), q(p + "mlp.up_proj.weight")),
                                    wdown=q(p + "mlp.down_proj.weight"), g1=g1, g2=g2))
        self._nf4_ready()
        return self

    def _nf4_ready(self):
        self._graphs = {}
        # decode at batch > NF4_MAX_M dequantises into a workspace whose address a captured graph keeps: size it now
        if self.device.type == "cuda" and self.max_batch > ops.NF4_MAX_M:
            ops.reserve_nf4_workspace([w for L in self.layers for w in (L["wqkv"], L["wo"], L["wgu"], L["wdown"])],
                                      self.device)

    @property
    def nf4(self):
        return bool(self.layers) and isinstance(self.layers[0]["wqkv"], _nf4.NF4Weight)

    def init_random(self, seed=0, std=0.02, nf4=False):
        """Random-init weights of the configured architecture directly on the device (benchmarks); nf4=True quantises
        the projections as load_state_dict(nf4=True) does (unit RMSNorm gains, applied as the column scale)."""
        c, dev = self.cfg, self.device
        g = torch.Generator(device=dev).manual_seed(seed)

        def w(*shape):
            v = (torch.randn(shape, generator=g, device=dev, dtype=torch.float32) * std).to(BF16)
            return _nf4.quantize(v) if nf4 and len(shape) == 2 and shape != (c.vocab_size, c.hidden_size) else v

        self.embed = w(c.vocab_size, c.hidden_size)
        self.lm_head = w(c.vocab_size, c.hidden_size)  # unit RMSNorm gains: folding is the identity
        self.layers = []
        ones = torch.ones((c.hidden_size,), dtype=torch.float32, device=dev)
        for _ in range(c.num_hidden_layers):
            gate, up = w(c.intermediate_size, c.hidden_size), w(c.intermediate_size, c.hidden_size)
            L = dict(wqkv=w(3 * c.hidden_size, c.hidden_size), wo=w(c.hidden_size, c.hidden_size),
                     wgu=_pack_glu_nf4(gate, up) if nf4 else ops.pack_glu_weight(gate, up),
                     wdown=w(c.hidden_size, c.intermediate_size))
            if nf4:
                L.update(g1=ones, g2=ones)
            self.layers.append(L)
        if nf4:
            self._nf4_ready()
        self._graphs = {}
        return self

    def state_dict(self, prefix=""):
        """Reference-named tensors (HF LlamaForCausalLM names, bf16) rebuilt from the packed device weights: q/k/v and
        gate/up are un-fused, the folded RMSNorm gains divided out again (exact where the gain is 1, else within one
        bf16 rounding of the loaded value)."""
        c, out = self.cfg, {}
        d, f = c.hidden_size, c.intermediate_size
        gains = getattr(self, "norm_gains", None)
        ones = torch.ones((d,), dtype=torch.float32, device=self.device)
        nf4 = self.nf4

        def unfold(w, g):
            # NF4 layers hold the unfolded W_eff (returned in bf16; bitsandbytes' packed-uint8 state dict is not reproduced)
            if isinstance(w, _nf4.NF4Weight):
                return _nf4.dequantize(w).to(BF16)
            return (w.float() / g[None, :]).to(BF16)
        out[prefix + "model.embed_tokens.weight"] = self.embed
        gn = gains["norm"] if gains else ones
        out[prefix + "model.norm.weight"] = gn.to(BF16)
        out[prefix + "lm_head.weight"] = unfold(self.lm_head, gn)
        for i, L in enumerate(self.layers):
            p = f"{prefix}model.layers.{i}."
            g1 = gains["ln1"][i] if gains else ones
            g2 = gains["ln2"][i] if gains else ones
            q, k, v = (L["wqkv"].rows(j * d, (j + 1) * d) for j in range(3)) if nf4 else L["wqkv"].split(d, 0)
            out[p + "self_attn.q_proj.weight"], out[p + "self_attn.k_proj.weight"], out[p + "self_attn.v_proj.weight"] = \
                unfold(q, g1), unfold(k, g1), unfold(v, g1)
            dense = lambda w: _nf4.dequantize(w).to(BF16) if nf4 else w
            out[p + "self_attn.o_proj.weight"] = dense(L["wo"])
            wgu = _nf4.dequantize(L["wgu"]) if nf4 else L["wgu"]
            gu = wgu.view(f // 16, 2, 16, d)           # ops.pack_glu_weight: 16-row blocks [gate | up]
            out[p + "mlp.gate_proj.weight"] = unfold(gu[:, 0].reshape(f, d), ones if nf4 else g2)
            out[p + "mlp.up_proj.weight"] = unfold(gu[:, 1].reshape(f, d), ones if nf4 else g2)
            out[p + "mlp.down_proj.weight"] = dense(L["wdown"])
            out[p + "input_layernorm.weight"] = g1.to(BF16)
            out[p + "post_attention_layernorm.weight"] = g2.to(BF16)
        return out

    def parameters(self):
        yield self.embed
        yield self.lm_head
        for L in self.layers:
            for w in (L["wqkv"], L["wo"], L["wgu"], L["wdown"]):
                if isinstance(w, _nf4.NF4Weight):
                    yield from (w.codes, w.scales)
                else:
                    yield w

    def weight_bytes(self):
        """Bytes of weights one decode step streams (lm_head and the layer projections; NF4 codes + scales as stored)."""
        n = 2 * self.lm_head.numel()
        for l in self.layers:
            for w in (l["wqkv"], l["wo"], l["wgu"], l["wdown"]):
                n += w.nbytes if isinstance(w, _nf4.NF4Weight) else 2 * w.numel()
        return n

    # ------------------------------------------------------------------ layers
    def _layer(self, i, h, positions, bot, slots, prefill_shape=None, kv_len=None, max_kv_len=0, q_start=None,
               beam=False):
        """h [T, d] is updated in place and returned. RMSNorm is never a kernel of its own: its gain is
        folded into wqkv / wgu and 1/rms is a row scale of the GEMM epilogue (computed inside the
        weight-streaming kernel for T <= 16). With q_start (append) the chunk attends over the paged cache: kv_len is
        then the chunk length per row and max_kv_len the longest cached + chunk length."""
        c, L, cache = self.cfg, self.layers[i], self.cache
        H, D = c.num_attention_heads, c.head_dim
        g1, g2 = L.get("g1"), L.get("g2")        # RMSNorm gains of NF4 layers (bf16 layers have them folded in)
        qkv = ops.gemm(h, L["wqkv"], rms_eps=c.rms_norm_eps, **({} if g1 is None else dict(kscale=g1)))
        if prefill_shape is not None:
            B, S = prefill_shape
            ops.rope_kv_append(qkv, positions, H, D, c.rope_theta, cache.k(i), cache.v(i), cache.block_table, bot, slots,
                               cache.page_size)
            q4 = qkv.view(B, S, 3, H, D)
            if q_start is None:
                att = ops.attention(q4[:, :, 0], q4[:, :, 1], q4[:, :, 2], causal=True, kv_len=kv_len)
            else:   # the chunk's K / V were just scattered to their pages: every key is read from the cache
                att = ops.attention_paged(q4[:, :, 0], cache.k(i), cache.v(i), cache.block_table[:B], q_start, kv_len,
                                          max_kv_len)
            att = att.view(B * S, H * D)
        elif beam:   # beam rows read their generated keys through the beam indirection
            T = h.shape[0]
            att = ops.attn_decode_rope_beam(qkv, self._rope_tab, cache.k(i), cache.v(i), cache.block_table, kv_len,
                                            self.beam["beam_src"][:T], self.d_prompt[:T], H, D, cache.page_size,
                                            max_kv_len)
        else:  # decode: RoPE + KV append happen inside the attention kernel
            att = ops.attn_decode_rope(qkv, self._rope_tab, cache.k(i), cache.v(i), cache.block_table, kv_len, H, D,
                                       cache.page_size, max_kv_len)
        ops.gemm(att, L["wo"], residual=h, out=h)
        act = ops.gemm(h, L["wgu"], glu=ops.GLU_SWIGLU, rms_eps=c.rms_norm_eps, **({} if g2 is None else dict(kscale=g2)))
        ops.gemm(act, L["wdown"], residual=h, out=h)
        return h

    # ------------------------------------------------------------------ prefill
    def prefill(self, inputs_embeds, seq_lens=None, all_logits=False):
        """inputs_embeds [B, S, d] bf16 (right padded), seq_lens list/tensor of valid lengths.
        Fills the KV cache for slots 0..B-1 and returns fp32 logits of the last valid token [B, V]
        (or of every position [B, S, V] when all_logits)."""
        c, dev, cache = self.cfg, self.device, self.cache
        B, S, d = inputs_embeds.shape
        if B > self.max_batch:
            raise ValueError(f"batch {B} > engine max_batch {self.max_batch}")
        lens = [S] * B if seq_lens is None else [int(x) for x in seq_lens]
        if max(lens) > cache.max_seq_len or S > cache.max_seq_len:
            # the K/V scatter indexes block_table[b, slot // page_size]: a prompt longer than the table must never launch
            raise ValueError(f"prompt of {max(max(lens), S)} tokens exceeds the KV cache capacity {cache.max_seq_len} "
                             f"(construct the model with a larger max_seq_len)")
        for b in range(self.max_batch):
            cache.release(b)
        for b in range(B):
            cache.reserve(b, lens[b])
        cache.sync_table()
        ar = torch.arange(S, dtype=torch.int32)
        lens_t = torch.tensor(lens, dtype=torch.int32)
        pos_h = ar.repeat(B)
        valid = (ar[None, :] < lens_t[:, None]).reshape(-1)
        slots_h = torch.where(valid, pos_h, torch.full_like(pos_h, -1))
        bot_h = torch.arange(B, dtype=torch.int32).repeat_interleave(S)
        positions = pos_h.to(dev, non_blocking=True)
        slots = slots_h.to(dev, non_blocking=True)
        bot = bot_h.to(dev, non_blocking=True)
        kv_len = lens_t.to(dev, non_blocking=True)
        h = inputs_embeds.to(BF16).reshape(B * S, d).clone()
        for i in range(c.num_hidden_layers):
            self._layer(i, h, positions, bot, slots, prefill_shape=(B, S), kv_len=kv_len)
        # decode state: next token goes to position / slot P, attention then spans P + 1 keys
        self.d_pos[:B].copy_(kv_len)
        self.d_len[:B].copy_(kv_len + 1)
        self.d_prompt[:B].copy_(kv_len)
        self._lens_host = list(lens)
        if all_logits:
            return ops.gemm(h, self.lm_head, out_fp32=True, rms_eps=c.rms_norm_eps).view(B, S, c.vocab_size)
        last = (torch.arange(B) * S + (lens_t.long() - 1)).to(dev)
        hl = h.index_select(0, last)
        return ops.gemm(hl, self.lm_head, out_fp32=True, rms_eps=c.rms_norm_eps)

    # ------------------------------------------------------------------ append
    def append(self, inputs_embeds, chunk_lens, all_logits=True, past_lens=None):
        """Extend the cached sequences of slots 0..B-1 by a chunk: inputs_embeds [B, S, d] bf16 (right padded),
        chunk_lens = valid tokens per row. past_lens (default: the lengths the last prefill / append left) = cached
        tokens each row continues from; positions at or past it are overwritten, so appending twice from the same past
        branches. Returns fp32 logits of every chunk position [B, S, V] (or of the last valid one [B, V])."""
        c, dev, cache = self.cfg, self.device, self.cache
        B, S, d = inputs_embeds.shape
        if B > self.max_batch:
            raise ValueError(f"batch {B} > engine max_batch {self.max_batch}")
        past = list(self._lens_host[:B]) if past_lens is None else [int(x) for x in past_lens]
        lens = [int(x) for x in chunk_lens]
        if len(past) != B or len(lens) != B or min(lens) < 1 or max(lens) > S or min(past) < 0:
            raise ValueError(f"chunk lengths {lens} / past lengths {past} do not fit a [{B}, {S}] chunk")
        total = [p + n for p, n in zip(past, lens)]
        if max(total) > cache.max_seq_len:
            raise ValueError(f"prompt of {max(total)} tokens exceeds the KV cache capacity {cache.max_seq_len} "
                             f"(construct the model with a larger max_seq_len)")
        changed = False
        for b in range(B):
            changed |= cache.reserve(b, total[b])
        if changed:
            cache.sync_table()
        ar = torch.arange(S, dtype=torch.int32)
        past_t, lens_t = torch.tensor(past, dtype=torch.int32), torch.tensor(lens, dtype=torch.int32)
        pos_h = (past_t[:, None] + ar[None, :]).reshape(-1)
        valid = (ar[None, :] < lens_t[:, None]).reshape(-1)
        slots_h = torch.where(valid, pos_h, torch.full_like(pos_h, -1))      # -1: padding, the K/V scatter skips it
        bot_h = torch.arange(B, dtype=torch.int32).repeat_interleave(S)
        positions, slots, bot = (t.to(dev, non_blocking=True) for t in (pos_h, slots_h, bot_h))
        q_start, q_len = past_t.to(dev, non_blocking=True), lens_t.to(dev, non_blocking=True)
        h = inputs_embeds.to(BF16).reshape(B * S, d).clone()
        for i in range(c.num_hidden_layers):
            self._layer(i, h, positions, bot, slots, prefill_shape=(B, S), kv_len=q_len, max_kv_len=max(total),
                        q_start=q_start)
        # decode state continues after the chunk, as after a prefill of the whole sequence
        tot_t = torch.tensor(total, dtype=torch.int32).to(dev, non_blocking=True)
        self.d_pos[:B].copy_(tot_t)
        self.d_len[:B].copy_(tot_t + 1)
        self.d_prompt[:B].copy_(tot_t)
        self._lens_host = list(total)
        if all_logits:
            return ops.gemm(h, self.lm_head, out_fp32=True, rms_eps=c.rms_norm_eps).view(B, S, c.vocab_size)
        last = (torch.arange(B) * S + (lens_t.long() - 1)).to(dev)
        return ops.gemm(h.index_select(0, last), self.lm_head, out_fp32=True, rms_eps=c.rms_norm_eps)

    # ------------------------------------------------------------------ decode
    def _decode_body(self, B, beam=False):
        """One greedy token for slots 0..B-1: reads d_src/d_pos/d_len, leaves logits in d_logits,
        arg-max in d_next, and advances the device-side counters."""
        c = self.cfg
        h = ops.splice_multimodal(self.embed, None, self.d_src[:B])
        self._rope_tab = ops.rope_table(self.d_pos[:B], c.head_dim, c.rope_theta, out=self.d_rope[:B])
        for i in range(c.num_hidden_layers):
            self._layer(i, h, self.d_pos[:B], self.d_bot[:B], None, kv_len=self.d_len[:B],
                        max_kv_len=self.cache.max_seq_len, beam=beam)
        ops.gemm(h, self.lm_head, out=self.d_logits[:B], out_fp32=True, rms_eps=c.rms_norm_eps)

    def _step_kernels(self, B, sampled=False):
        from . import _lib
        lib = _lib.load()
        prev = lib.vb200_set_pdl(1 if self.use_pdl else 0)  # decode-step kernels overlap via PDL
        try:
            self._step_kernels_inner(B, sampled)
        finally:
            lib.vb200_set_pdl(prev)

    def _step_kernels_inner(self, B, sampled=False):
        if sampled in ("beam", "beam_sample"):
            self._decode_body(B, beam=True)
            if self.proc_on:
                self.process_logits(self.d_logits[:B], step=True, beam=True)
            self.beam_advance(self.d_logits[:B], sample=sampled == "beam_sample", logprobs=self.proc_on)
            return
        self._decode_body(B)
        if self.proc_on:
            self.process_logits(self.d_logits[:B], step=True)
        # token_log[b, d_len - d_prompt] = token; d_src = token; d_pos += 1; d_len += 1
        state = dict(next_src=self.d_src[:B], positions=self.d_pos[:B], kv_len=self.d_len[:B], token_log=self.token_log[:B],
                     prompt_len=self.d_prompt[:B])
        if sampled:
            self.sample_advance(self.d_logits[:B], self.d_next[:B], **state)
        else:
            ops.argmax_advance(self.d_logits[:B], self.d_next[:B], **state)

    def sample_advance(self, logits, out_idx=None, **state):
        """Sample rows of fp32 logits with the set_sampling parameters (ops.sample_advance arguments after `params`).
        A CUDA engine runs the kernel; a CPU engine, which runs no kernels of this library, runs the host statement of
        the same contract (vitron_b200.sampling)."""
        fn = ops.sample_advance if self.device.type == "cuda" else sampling.sample_advance
        return fn(logits, self.d_sample, out_idx, **state)

    def set_sampling(self, temperature=1.0, top_k=None, top_p=None, seed=0):
        """Parameters of the sampled decode step (read from self.d_sample): temperature clamped to >= 1e-6,
        top_k None / 0 = off, top_p None = off, 64-bit Philox seed."""
        k = 0 if not top_k or top_k < 0 else min(int(top_k), 2 ** 31 - 1)
        p = 1.0 if top_p is None else float(top_p)
        self.d_sample.copy_(ops.sample_params(max(float(temperature), 1e-6), k, p, seed))

    def set_processors(self, prompt_ids, repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0,
                       eos_ids=()):
        """Turn on the HF 4.31 logits processors (vitron_b200.processors) for the next decode: prompt_ids [R, input_len]
        are the raw input_ids of engine rows 0..R-1 (a beam row gets its request's row), eos_ids the EOS ids the
        minimum-length rules ban. The settings follow 4.31's enable rules; with none enabled the processors are off.
        The step reads them from device buffers, so new settings replay the captured graphs."""
        settings, on = processors.check_settings(repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens,
                                                 list(eos_ids))
        if not on:
            return self.clear_processors()
        R, n_in = prompt_ids.shape
        S = self.cache.max_seq_len
        if R > self.max_batch:
            raise ValueError(f"{R} prompt rows > engine max_batch {self.max_batch}")
        if n_in > S or 2 * S > processors.MAX_HIST:
            raise ValueError(f"logits processors stage at most {processors.MAX_HIST} history tokens per row: an input of "
                             f"{n_in} columns on an engine of max_seq_len {S} does not fit")
        eos = list(eos_ids) if settings["min_length"] or settings["min_new_tokens"] else []
        self.d_proc.copy_(processors.pack_params(input_len=n_in, eos_ids=eos, **settings))
        self.d_proc_prompt[:R, :n_in].copy_(prompt_ids.to(torch.int32))
        self.proc_on = True

    def clear_processors(self):
        self.proc_on = False

    def process_logits(self, logits, step=False, beam=False):
        """Apply the set_processors settings in place to rows of fp32 logits: step=False is the first generated token
        (the prefill logits, nothing generated yet); step=True a decode step, reading the rows' generated ids from
        token_log (through beam_src for beam rows, which get log-softmax first). A CUDA engine runs the kernel; a CPU
        engine runs the host statement of the same contract (vitron_b200.processors)."""
        R = logits.shape[0]
        state = {}
        if step:
            state = dict(token_log=self.token_log[:R], kv_len=self.d_len[:R], prompt_len=self.d_prompt[:R])
            if beam:
                state["beam_src"] = self.beam["beam_src"][:R]
        fn = ops.logits_process if self.device.type == "cuda" else processors.process
        return fn(logits, self.d_proc, self.d_proc_prompt[:R], logprobs=beam, **state)

    def _beam_state(self):
        if self.beam is None:
            R, S, dev = self.max_batch, self.cache.max_seq_len, self.device
            z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt, device=dev)
            self.beam = dict(beam_score=z(R, dt=torch.float32), parent=z(R), done=z(R), beam_src=z(R, S),
                             hyp_score=z(R, dt=torch.float64), hyp_len=z(R), hyp_seq=z(R), hyp_count=z(R),
                             hyp_ids=z(R, S, dt=torch.int64))
            self.d_beam = torch.zeros((_beam.PARAMS.size,), dtype=torch.uint8, device=dev)
            if dev.type == "cuda":
                ops.reserve_beam_workspace(R, dev)
        return self.beam

    def _require_beam(self):
        if self.beam is None or self.beam_k < 1:
            raise RuntimeError("no beam search is set up on this engine: call start_beam() before beam steps")

    def beam_advance(self, logits, sample=False, logprobs=False):
        """The beam step over rows of fp32 logits with the start_beam parameters (sample=True: the beam-sampling step,
        with the set_sampling parameters too; logprobs=True: the rows hold processed log-probabilities). A CUDA engine
        runs the kernel; a CPU engine, which runs no kernels of this library, runs the host statement of the same
        contract (vitron_b200.beam)."""
        self._require_beam()
        R = logits.shape[0]
        state = dict({n: t[:R] for n, t in self.beam.items()}, next_src=self.d_src[:R], positions=self.d_pos[:R],
                     kv_len=self.d_len[:R], token_log=self.token_log[:R], prompt_len=self.d_prompt[:R])
        if sample:
            fn = ops.beam_sample_advance if self.device.type == "cuda" else _beam.beam_sample_advance
            fn(logits, self.beam_k, self.d_beam, self.d_sample, **state, logprobs=logprobs)
        else:
            fn = ops.beam_advance if self.device.type == "cuda" else _beam.beam_advance
            fn(logits, self.beam_k, self.d_beam, **state, logprobs=logprobs)

    def start_beam(self, logits, k, max_new_tokens, params, sample=False, searches=1):
        """Beam search over the B prompts of the last prefill: logits [B, V] are its last-token logits, params a
        beam.pack_params buffer. Rows b * k + j become the beams of request b, sharing its full prompt pages (the partial
        last page is copied per beam); step 0 runs the beam kernel on the logits replicated to the k rows (generated
        token 0). decode_steps(B * k, n, sampled="beam") then runs further steps.

        sample=True is beam sampling with the set_sampling parameters (decode_steps(..., sampled="beam_sample")), every
        beam starting at score 0, and
        searches = r runs r independent searches per prompt: search b * r + i (rows (b * r + i) * k + j) samples prompt
        b, so the prompt's pages are shared by r * k rows."""
        B = logits.shape[0]
        R, lens = B * searches * k, [int(x) for x in self._lens_host[:B]]
        if not 1 <= k <= _beam.MAX_K:
            raise ValueError(f"num_beams must be in 1..{_beam.MAX_K}, got {k}")
        if searches < 1:
            raise ValueError(f"searches must be >= 1, got {searches}")
        if R > self.max_batch:
            raise ValueError(f"batch {B} x {searches} searches x num_beams {k} = {R} rows > engine max_batch "
                             f"{self.max_batch}")
        need = max(lens) + max_new_tokens
        if need > self.cache.max_seq_len:
            raise ValueError(f"prompt + max_new_tokens = {need} exceeds KV capacity {self.cache.max_seq_len}")
        st = self._beam_state()
        self.cache.fork(lens, searches * k)
        rk = searches * k
        for r in range(R):
            self.cache.reserve(r, lens[r // rk] + max_new_tokens)
        self.cache.sync_table()
        self.beam_k = k
        self.d_beam.copy_(params)
        plen = torch.tensor(lens, dtype=torch.int32).repeat_interleave(rk).to(self.device)
        self.d_prompt[:R].copy_(plen)
        self.d_len[:R].copy_(plen)            # kv_len - prompt_len = 0: the step below logs generated token 0
        self.d_pos[:R].copy_(plen - 1)
        self._lens_host = plen.tolist()
        init = torch.full((B * searches, k), -1e9, dtype=torch.float32)
        init[:, 0] = 0.0
        if sample:              # 4.31 beam_sample starts every beam at 0 (beam_search starts beams 1..k-1 at -1e9)
            init.zero_()
        st["beam_score"][:R].copy_(init.reshape(-1))
        for name in ("done", "hyp_count"):
            st[name][:B * searches].zero_()
        rows = logits.float().repeat_interleave(rk, 0).contiguous()
        if self.proc_on:     # the first generated token: the processors see the prompt only
            self.process_logits(rows, beam=True)
        self.beam_advance(rows, sample=sample, logprobs=self.proc_on)

    def start_decode(self, first_tokens, max_new_tokens):
        """first_tokens [B] int64: the token chosen from the prefill logits (already counted as
        generated token 0). Prepares device state for up to max_new_tokens-1 further steps."""
        B = first_tokens.shape[0]
        dev = self.device
        need = max(int(x) for x in self._lens_host) + max_new_tokens
        if need > self.cache.max_seq_len:
            raise ValueError(f"prompt + max_new_tokens = {need} exceeds KV capacity {self.cache.max_seq_len}")
        changed = False
        for b in range(B):
            changed |= self.cache.reserve(b, self._lens_host[b] + max_new_tokens)
        if changed:
            self.cache.sync_table()
        self.token_log[:B, 0] = first_tokens
        self.d_src[:B] = first_tokens.to(torch.int32)

    def decode_steps(self, B, n, use_graph=True, sampled=False):
        """Run n decode steps for slots 0..B-1 (no host sync): greedy, sampled with the set_sampling parameters, or
        (sampled="beam" / "beam_sample") beam-search / beam-sampling steps over the B = searches x num_beams rows of
        start_beam. The beam modes read their parameters from device buffers: one graph per (rows, mode, k). The logits
        processors (set_processors) also read theirs from device buffers: one graph more per key with them on."""
        if n <= 0:
            return
        beam_mode = sampled in ("beam", "beam_sample")
        if beam_mode:
            self._require_beam()
        if not use_graph or self.device.type != "cuda":   # (host-logic tests drive the same step un-graphed)
            for _ in range(n):
                self._step_kernels(B, sampled)
            return
        key = (B, sampled, self.beam_k, self.proc_on) if beam_mode else (B, bool(sampled), self.proc_on)
        if key not in self._graphs:
            # warm-up on a side stream (allocator + lazy init), then capture
            s = torch.cuda.Stream(device=self.device)
            s.wait_stream(torch.cuda.current_stream())
            state = [self.d_src, self.d_pos, self.d_len, self.token_log]
            if beam_mode:
                state += list(self.beam.values())
            saved = [t.clone() for t in state]
            with torch.cuda.stream(s):
                self._step_kernels(B, sampled)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            for t, sv in zip(state, saved):
                t.copy_(sv)
            g = torch.cuda.CUDAGraph()
            l0 = ops.launch_count()
            with torch.cuda.graph(g):
                self._step_kernels(B, sampled)
            for t, sv in zip(state, saved):
                t.copy_(sv)
            self._graphs[key] = (g, ops.launch_count() - l0)
        g, self.launches_per_step = self._graphs[key]     # graphs with processors launch one kernel more
        for _ in range(n):
            g.replay()
        ops.count_launches(n * self.launches_per_step)

    def decode_one_logits(self, tokens):
        """Teacher forcing: feed tokens [B] and return fp32 logits [B, V] (the next token is the caller's choice)."""
        B = tokens.shape[0]
        self.d_src[:B] = tokens.to(torch.int32)
        self._decode_body(B)
        self.d_pos[:B].add_(1)
        self.d_len[:B].add_(1)
        return self.d_logits[:B]


def _pack_glu_nf4(a, b):
    """ops.pack_glu_weight's 16-row interleave applied to the rows of two NF4 weights."""
    return _nf4.NF4Weight(ops.pack_glu_weight(a.codes, b.codes), ops.pack_glu_weight(a.scales, b.scales), a.k)
