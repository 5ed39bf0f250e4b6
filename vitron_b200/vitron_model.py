"""VitronLlamaForCausalLM — drop-in for the reference's LlavaLlamaForCausalLM on H100 kernels.

Mirrors vitron/model/language_model/llava_llama.py:40-114 (`forward`, `generate` via HF
GenerationMixin, `prepare_inputs_for_generation`) and vitron/model/llava_arch.py:153-573
(`encode_images`, `encode_videos`, `prepare_inputs_labels_for_multimodal`) — same method names,
argument meaning, sentinel handling (IMAGE_TOKEN_INDEX -200, OBJS_TOKEN_INDEX -300), truncation and
padding rules, and the reference's parameter names for `load_state_dict`.

Mechanism: the per-sample Python cat/split loop becomes one host-side layout pass over the (tiny)
id tensor plus a single gather kernel; the decoder runs on `LlamaEngine` (paged KV cache, fused
kernels, CUDA-graph decode, arg-max or sampler on device).
"""
from types import SimpleNamespace

import torch

from . import beam, ops, processors
from .module_face import ModuleFace
from .adapters import RegionExtractor, VisionProjector
from .llama import LlamaConfig, LlamaEngine
from .vision_tower import LanguageBindImageTower, LanguageBindVideoTower, VisionConfig

BF16 = torch.bfloat16
IGNORE_INDEX = -100          # vitron/constants.py:7
IMAGE_TOKEN_INDEX = -200     # vitron/constants.py:9
OBJS_TOKEN_INDEX = -300      # vitron/constants.py:24
PAD_SRC = -2147483648


def layout_multimodal(ids_h, mask_h, labels_h, feat_rows, region_rows, max_model_len, left_pad):
    """Host half of prepare_inputs_labels_for_multimodal (vitron/model/llava_arch.py:300-372, 470-556).

    ids_h / mask_h / labels_h: CPU [B, L]; feat_rows[e]: rows of image-feature entry e (video frames are
    separate entries); region_rows[e]: rows of its region feature or None (None list = no regions).
    Returns (srcmap int32 [B, S], labels [B, S], attention_mask bool [B, S], position_ids [B, S], lens):
    srcmap >= 0 -> token id, -(row+1) -> row of the concatenated [features ; region features] buffer,
    INT32_MIN -> padding. Quirks kept: a sample without <image> consumes one feature slot (:492); an
    <objs> token takes the region feature of the most recent image (index cur-1, Python-negative for
    cur == 0)."""
    use_regions = region_rows is not None
    feat_base, off = [], 0
    for n in feat_rows:
        feat_base.append(off)
        off += n
    region_slot = {}
    if use_regions:
        for e, n in enumerate(region_rows):
            if n is not None:
                region_slot[e] = off
                off += n
    srcs, labs = [], []
    cur = 0
    for b in range(ids_h.shape[0]):
        ids_b = ids_h[b][mask_h[b]].tolist()
        lab_b = labels_h[b][mask_h[b]].tolist()
        n_img = sum(1 for t in ids_b if t == IMAGE_TOKEN_INDEX)
        src, lab = [], []
        if n_img == 0:
            if any(t < 0 for t in ids_b):
                raise ValueError("special sentinel in a sample without <image> tokens")
            src, lab = list(ids_b), list(lab_b)
            cur += 1
        else:
            for t, l in zip(ids_b, lab_b):
                if t == IMAGE_TOKEN_INDEX:
                    if cur >= len(feat_rows):
                        raise IndexError("more <image> tokens than images")
                    src.extend(-(feat_base[cur] + i) - 1 for i in range(feat_rows[cur]))
                    lab.extend([IGNORE_INDEX] * feat_rows[cur])
                    cur += 1
                elif t == OBJS_TOKEN_INDEX:
                    if not use_regions:
                        raise ValueError("<objs> token given but no regions")
                    e = (cur - 1) % len(feat_rows)
                    if e not in region_slot:
                        raise ValueError("region feature requested for a video frame")
                    src.extend(-(region_slot[e] + i) - 1 for i in range(region_rows[e]))
                    lab.extend([IGNORE_INDEX] * region_rows[e])
                else:
                    src.append(t)
                    lab.append(l)
        srcs.append(src)
        labs.append(lab)
    if max_model_len is not None:
        srcs = [s[:max_model_len] for s in srcs]
        labs = [l[:max_model_len] for l in labs]
    max_len = max(len(s) for s in srcs)
    B = len(srcs)
    src_t = torch.full((B, max_len), PAD_SRC, dtype=torch.int32)
    lab_t = torch.full((B, max_len), IGNORE_INDEX, dtype=labels_h.dtype)
    am = torch.zeros((B, max_len), dtype=torch.bool)
    pid = torch.zeros((B, max_len), dtype=torch.long)
    for b, (s, l) in enumerate(zip(srcs, labs)):
        n = len(s)
        if n == 0:
            continue
        sl = slice(max_len - n, max_len) if left_pad else slice(0, n)
        src_t[b, sl] = torch.tensor(s, dtype=torch.int32)
        lab_t[b, sl] = torch.tensor(l, dtype=labels_h.dtype)
        am[b, sl] = True
        pid[b, sl] = torch.arange(n)
    return src_t, lab_t, am, pid, [len(s) for s in srcs]


class VitronConfig(SimpleNamespace):
    def __init__(self, llm=None, vision=None, video=None, mm_projector_type="mlp2x_gelu",
                 mm_vision_select_layer=-2, mm_vision_select_feature="patch", tokenizer_padding_side="right",
                 tokenizer_model_max_length=None, pad_token_id=0, eos_token_id=2, bos_token_id=1, **kw):
        llm = LlamaConfig.from_any(llm or {})
        vision = vision if isinstance(vision, VisionConfig) or vision is None else VisionConfig(**vision)
        video = video if isinstance(video, VisionConfig) or video is None else VisionConfig(**video)
        super().__init__(llm=llm, vision=vision, video=video, mm_projector_type=mm_projector_type,
                         mm_vision_select_layer=mm_vision_select_layer,
                         mm_vision_select_feature=mm_vision_select_feature,
                         tokenizer_padding_side=tokenizer_padding_side,
                         tokenizer_model_max_length=tokenizer_model_max_length, pad_token_id=pad_token_id,
                         eos_token_id=eos_token_id, bos_token_id=bos_token_id,
                         hidden_size=llm.hidden_size, vocab_size=llm.vocab_size,
                         mm_hidden_size=(vision or video).hidden_size if (vision or video) else 0, **kw)


class _InnerModel:
    """Stands in for `LlavaLlamaModel` (get_model()): owns towers, projector, region extractor."""

    def __init__(self):
        self.image_tower = None
        self.video_tower = None
        self.mm_projector = None
        self.region_extractor = None
        self.engine = None

    def get_image_tower(self):
        return self.image_tower

    def get_video_tower(self):
        return self.video_tower

    def get_region_extractor(self):
        return self.region_extractor

    def embed_tokens(self, ids):
        src = ids.to(device=self.engine.device, dtype=torch.int32).contiguous()
        return ops.splice_multimodal(self.engine.embed, None, src)


class CausalLMOutput(SimpleNamespace):
    pass


class PagedPast:
    """`past_key_values` of VitronLlamaForCausalLM.forward: a handle on the rows of the engine's paged KV cache, not a
    copy. `lens[b]` = tokens cached for row b (image features counted as the positions they fill), `seq_len` = the
    longest. `len(past)` is the layer count and `past[layer]` gathers that layer's (k, v) as [B, H, seq_len, head_dim]
    copies (row b's keys at [0, lens[b]), zeros after), so reference code such as `past[-1][-1].shape[-2]` works.

    A handle stays usable while the cache positions it covers are intact: appending from it (even twice: branching)
    keeps it valid; generate(), a forward without past_key_values, or an append from a shorter handle that overwrote
    positions below its length make it stale, and using a stale handle raises ValueError."""

    def __init__(self, model, lens, segments):
        self._model, self.lens, self._segments = model, list(lens), segments

    @property
    def seq_len(self):
        return max(self.lens)

    def __len__(self):
        return self._model.engine.cfg.num_hidden_layers

    def __getitem__(self, layer):
        self._model._check_past(self)
        eng = self._model.engine
        cache, c = eng.cache, eng.cfg
        i = range(c.num_hidden_layers)[layer]
        B, S = len(self.lens), self.seq_len
        out = []
        for pages in (cache.k(i), cache.v(i)):
            t = torch.zeros((B, c.num_attention_heads, S, c.head_dim), dtype=pages.dtype, device=pages.device)
            for b, n in enumerate(self.lens):
                idx = torch.tensor(cache._owned[b][:(n + cache.page_size - 1) // cache.page_size], dtype=torch.long,
                                   device=pages.device)
                t[b, :, :n] = pages[idx].permute(1, 0, 2, 3).reshape(c.num_attention_heads, -1, c.head_dim)[:, :n]
            out.append(t)
        return tuple(out)


class VitronLlamaForCausalLM(ModuleFace):
    def __init__(self, config, device="cuda", max_batch=8, max_seq_len=2048):
        self.config = config
        self.device = torch.device(device)
        self.model = _InnerModel()
        self.model.engine = LlamaEngine(config.llm, self.device, max_batch=max_batch, max_seq_len=max_seq_len)
        sl, sf = config.mm_vision_select_layer, config.mm_vision_select_feature
        if config.vision is not None:
            self.model.image_tower = LanguageBindImageTower(config.vision, self.device, sl, sf)
        if config.video is not None:
            self.model.video_tower = LanguageBindVideoTower(config.video, self.device, sl, sf)
        if config.vision is not None or config.video is not None:
            vc = config.vision or config.video
            self.model.mm_projector = VisionProjector(config.mm_projector_type, vc.hidden_size,
                                                      config.llm.hidden_size, self.device)
            self.model.region_extractor = RegionExtractor(vc.hidden_size, config.llm.hidden_size, vc.patch_size,
                                                          vc.image_size, self.device)

    # ------------------------------------------------------------------ reference accessors
    def get_model(self):
        return self.model

    def get_image_tower(self):
        return self.model.get_image_tower()

    def get_video_tower(self):
        return self.model.get_video_tower()

    def get_region_extractor(self):
        return self.model.get_region_extractor()

    @property
    def engine(self):
        return self.model.engine

    def state_dict(self):
        """Reference-named tensors of everything this model owns (SURVEY.md Appendix B names)."""
        out = dict(self.engine.state_dict())
        m = self.model
        if m.mm_projector is not None:
            out.update(m.mm_projector.state_dict("model.mm_projector."))
        if m.region_extractor is not None and m.region_extractor.mlp:
            out.update(m.region_extractor.state_dict("model.region_extractor."))
        if m.image_tower is not None and m.image_tower.vit.layers:
            out.update(m.image_tower.vit.state_dict("model.image_tower.image_tower."))
        if m.video_tower is not None and m.video_tower.vit.layers:
            out.update(m.video_tower.vit.state_dict("model.video_tower.video_tower."))
        return out

    def parameters(self):
        yield from self.engine.parameters()
        m = self.model
        for sub in (m.mm_projector, m.region_extractor, m.image_tower, m.video_tower):
            if sub is not None:
                yield from sub.parameters()

    def resize_token_embeddings(self, new_num_tokens):
        """builder.py:146 `model.resize_token_embeddings(len(tokenizer))` after the special tokens were added: embedding and
        lm_head rows are appended (zeros: the reference's new rows are unseeded random values that inference never reads) or
        dropped; the decode state buffers follow the vocabulary."""
        eng = self.engine
        V, d = eng.embed.shape
        if new_num_tokens == V:
            return self
        def fit(w):
            out = torch.zeros((new_num_tokens, d), dtype=w.dtype, device=w.device)
            n = min(V, new_num_tokens)
            out[:n] = w[:n]
            return out
        eng.embed, eng.lm_head = fit(eng.embed), fit(eng.lm_head)
        eng.cfg.vocab_size = new_num_tokens
        eng.d_logits = torch.zeros((eng.max_batch, new_num_tokens), dtype=torch.float32, device=eng.device)
        eng._graphs = {}
        self.config.vocab_size = new_num_tokens
        return self

    def load_state_dict(self, sd, strict=True, nf4=False):
        """Accepts the reference's names: model.embed_tokens.*, model.layers.*, lm_head.weight,
        model.mm_projector.*, model.region_extractor.*, model.image_tower.image_tower.*,
        model.video_tower.video_tower.* (SURVEY.md Appendix B). nf4=True is the reference's load_4bit: the language
        model's projections, the mm_projector and the region extractor's Linears are NF4 (vitron_b200.nf4; bitsandbytes
        converts every Linear that LlavaMetaModel builds and skips only lm_head); the vision towers stay bf16."""
        self.engine.load_state_dict(sd, nf4=nf4)
        m = self.model
        if m.mm_projector is not None and any(k.startswith("model.mm_projector.") for k in sd):
            m.mm_projector.load_state_dict(sd, "model.mm_projector.", nf4=nf4)
        if m.region_extractor is not None and any(k.startswith("model.region_extractor.") for k in sd):
            m.region_extractor.load_state_dict(sd, "model.region_extractor.", nf4=nf4)
        if m.image_tower is not None and any(k.startswith("model.image_tower.image_tower.") for k in sd):
            m.image_tower.vit.load_state_dict(sd, "model.image_tower.image_tower.")
        if m.video_tower is not None and any(k.startswith("model.video_tower.video_tower.") for k in sd):
            m.video_tower.vit.load_state_dict(sd, "model.video_tower.video_tower.")
        return self

    # ------------------------------------------------------------------ encoders (llava_arch.py:168-187)
    def encode_images(self, images, regions=None):
        image_features = self.model.image_tower(images)
        region_features = None
        if regions is not None:
            region_features = self.model.region_extractor(image_features, regions)
        image_features = self.model.mm_projector(image_features)
        if region_features is not None:
            return image_features, region_features
        return image_features, torch.zeros_like(image_features)

    def encode_videos(self, videos):
        video_features = self.model.video_tower(videos)
        return self.model.mm_projector(video_features)

    # ------------------------------------------------------------------ splice (llava_arch.py:189-573)
    def prepare_inputs_labels_for_multimodal(self, input_ids, position_ids, attention_mask, past_key_values, labels,
                                             images, regions=None):
        image_tower, video_tower = self.get_image_tower(), self.get_video_tower()
        if (image_tower is None and video_tower is None) or images is None or input_ids.shape[1] == 1:
            if (past_key_values is not None and (image_tower is not None or video_tower is not None)
                    and images is not None and input_ids.shape[1] == 1):
                target = self._past_len(past_key_values) + 1
                attention_mask = torch.cat((attention_mask, torch.ones(
                    (attention_mask.shape[0], target - attention_mask.shape[1]), dtype=attention_mask.dtype,
                    device=attention_mask.device)), dim=1)
                position_ids = torch.sum(attention_mask, dim=1).unsqueeze(-1) - 1
            return input_ids, position_ids, attention_mask, past_key_values, None, labels

        use_regions = regions is not None and len(regions) > 0
        if isinstance(images, torch.Tensor):
            images = [im for im in images]
        image_idx = [i for i, im in enumerate(images) if im.ndim == 3]
        video_idx = [i for i, im in enumerate(images) if im.ndim == 4]
        feats = [None] * len(images)      # per entry: [n, d] tensor or list of T such tensors
        rfeats = [None] * len(images)
        if image_idx:
            mb = torch.stack([images[i] for i in image_idx]).to(self.device)
            rg = [regions[i] for i in image_idx] if use_regions else None
            f, r = self.encode_images(mb, rg)
            for j, pos in enumerate(image_idx):
                feats[pos] = f[j]
                rfeats[pos] = r[j] if use_regions else None
        if video_idx:
            vb = torch.stack([images[i] for i in video_idx]).to(self.device)
            vf = self.encode_videos(vb)  # [mb, t, n, d]
            for j, pos in enumerate(video_idx):
                feats[pos] = [vf[j, t] for t in range(vf.shape[1])]
                rfeats[pos] = [None] * vf.shape[1]
        flat, rflat = [], []
        for f, r in zip(feats, rfeats):
            if isinstance(f, list):
                flat.extend(f)
                rflat.extend(r)
            else:
                flat.append(f)
                rflat.append(r)

        # ---- host-side layout over the (tiny) id tensor: one D2H copy instead of the reference's
        # per-sample .sum()/.tolist() syncs (llava_arch.py:479-497)
        ids_h = input_ids.detach().cpu()
        _labels, _position_ids, _attention_mask = labels, position_ids, attention_mask
        mask_h = torch.ones_like(ids_h, dtype=torch.bool) if attention_mask is None else attention_mask.detach().cpu().bool()
        labels_h = torch.full_like(ids_h, IGNORE_INDEX) if labels is None else labels.detach().cpu()

        src_t, lab_t, am, pid, lens = layout_multimodal(
            ids_h, mask_h, labels_h, [f.shape[0] for f in flat],
            [None if r is None else r.shape[0] for r in rflat] if use_regions else None,
            getattr(self.config, "tokenizer_model_max_length", None),
            getattr(self.config, "tokenizer_padding_side", "right") == "left")

        pieces = [f.reshape(-1, f.shape[-1]) for f in flat]
        if use_regions:
            pieces += [r.reshape(-1, r.shape[-1]) for r in rflat if r is not None]
        feat_buf = torch.cat(pieces, 0).to(BF16).contiguous() if pieces else None
        inputs_embeds = ops.splice_multimodal(self.engine.embed, feat_buf, src_t.to(self.device))

        dev = input_ids.device
        new_labels = None if _labels is None else lab_t.to(dev)
        attention_mask = None if _attention_mask is None else am.to(device=dev, dtype=_attention_mask.dtype)
        position_ids = None if _position_ids is None else pid.to(dev)
        self._last_lens = lens
        return None, position_ids, attention_mask, past_key_values, inputs_embeds, new_labels

    @staticmethod
    def _past_len(past):
        if isinstance(past, int):
            return past
        if hasattr(past, "seq_len"):
            return past.seq_len
        return past[-1][-1].shape[-2]

    # ------------------------------------------------------------------ forward (llava_llama.py:57-102)
    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                inputs_embeds=None, labels=None, use_cache=None, output_attentions=None,
                output_hidden_states=None, images=None, regions=None, return_dict=None):
        """Logits for every position (fp32), like the reference. use_cache=True returns a PagedPast handle as
        `past_key_values`; passing it back appends the chunk (input_ids [B, n], attention_mask [B, past + n] that is 1
        over the chunk and whose past part sums to the handle's row lengths) to the cached rows and returns the chunk's
        logits [B, n, V] and a handle covering past + n. An image inside the chunk is spliced as in a first forward."""
        if past_key_values is not None:
            return self._forward_chunk(input_ids, attention_mask, past_key_values, inputs_embeds, labels, use_cache,
                                       images, regions)
        self._kv_segments = None          # the prefill below overwrites the cache: every handle becomes stale
        if inputs_embeds is None:
            if images is not None:
                (input_ids, position_ids, attention_mask, past_key_values, inputs_embeds, labels) = \
                    self.prepare_inputs_labels_for_multimodal(input_ids, position_ids, attention_mask,
                                                              past_key_values, labels, images, regions)
            if inputs_embeds is None:
                inputs_embeds = self.model.embed_tokens(input_ids)
        embeds, lens, restore = self._right_pad(inputs_embeds, attention_mask)
        logits = self.engine.prefill(embeds, lens, all_logits=True)
        if restore is not None:
            logits = restore(logits)
        past = self._new_past(lens, None) if use_cache else None
        return CausalLMOutput(loss=self._loss(logits, labels), logits=logits, past_key_values=past, hidden_states=None,
                              attentions=None)

    __call__ = forward

    @staticmethod
    def _loss(logits, labels):
        if labels is None:
            return None
        sl = logits[:, :-1].reshape(-1, logits.shape[-1])
        return torch.nn.functional.cross_entropy(sl, labels[:, 1:].reshape(-1).to(sl.device), ignore_index=IGNORE_INDEX)

    # ------------------------------------------------------------------ KV-cache handles
    # self._kv_segments[b] lists (end, write id) of the writes that produced cache positions [0, end) of row b; a handle
    # records the list its positions came from and is valid while that list is still a prefix of the current one.
    _kv_segments = None
    _kv_writes = 0

    def _new_past(self, lens, parent):
        self._kv_writes += 1
        w = self._kv_writes
        base = parent._segments if parent is not None else [[] for _ in lens]
        segs = [list(s) + [(n, w)] for s, n in zip(base, lens)]
        self._kv_segments = segs
        return PagedPast(self, lens, segs)

    def _check_past(self, past):
        if not isinstance(past, PagedPast):
            raise ValueError("past_key_values must be the PagedPast handle a forward(use_cache=True) of this model returned "
                             "(tuples of cache tensors are not accepted)")
        cur = self._kv_segments
        if (past._model is not self or cur is None or len(cur) != len(past._segments)
                or any(c[:len(s)] != s for c, s in zip(cur, past._segments))):
            raise ValueError("stale past_key_values: the KV cache positions it covers were overwritten since (generate(), "
                             "a forward without past_key_values, or an append from a shorter handle)")

    def _forward_chunk(self, input_ids, attention_mask, past, inputs_embeds, labels, use_cache, images, regions):
        self._check_past(past)
        B = len(past.lens)
        n = (input_ids if inputs_embeds is None else inputs_embeds).shape[1]
        if (input_ids if inputs_embeds is None else inputs_embeds).shape[0] != B:
            raise ValueError(f"chunk of {(input_ids if inputs_embeds is None else inputs_embeds).shape[0]} rows for a "
                             f"past of {B} rows")
        if attention_mask is not None:
            am = attention_mask.detach().cpu().bool()
            if am.shape[0] != B or am.shape[1] < n or not bool(am[:, am.shape[1] - n:].all()):
                raise ValueError(f"attention_mask must be [B, past + {n}] with ones over the chunk")
            if am[:, :am.shape[1] - n].sum(1).tolist() != past.lens:
                raise ValueError(f"the past part of attention_mask covers {am[:, :am.shape[1] - n].sum(1).tolist()} "
                                 f"tokens per row, the handle caches {past.lens}")
        chunk_mask = torch.ones((B, n), dtype=torch.long, device=(input_ids if inputs_embeds is None else inputs_embeds).device)
        am_chunk = None
        if inputs_embeds is None:
            if images is not None and n > 1:
                _, _, am_chunk, _, inputs_embeds, labels = self.prepare_inputs_labels_for_multimodal(
                    input_ids, None, chunk_mask, past, labels, images, regions)
            else:
                inputs_embeds = self.model.embed_tokens(input_ids)
        embeds, lens, restore = self._right_pad(inputs_embeds, am_chunk)
        logits = self.engine.append(embeds, lens, all_logits=True, past_lens=past.lens)
        if restore is not None:
            logits = restore(logits)
        total = [p + m for p, m in zip(past.lens, lens)]
        # the chunk's K / V now occupy positions past.lens.. of the cache whatever use_cache is: the write is recorded, so
        # that a handle whose positions it overwrote is seen as stale
        new_past = self._new_past(total, past)
        return CausalLMOutput(loss=self._loss(logits, labels), logits=logits,
                              past_key_values=new_past if use_cache is not False else None, hidden_states=None,
                              attentions=None)

    def _right_pad(self, embeds, attention_mask):
        """Engine wants right-padded rows. Returns (embeds, lens, restore_fn or None)."""
        B, S, _ = embeds.shape
        if attention_mask is None:
            return embeds, [S] * B, None
        am = attention_mask.bool().cpu()
        lens = am.sum(1).tolist()
        if all(bool(am[b, :lens[b]].all()) for b in range(B)):
            return embeds, lens, None
        # left padded (or holes): compact valid rows to the front, scatter results back afterwards
        idx = torch.zeros((B, S), dtype=torch.long)
        for b in range(B):
            v = torch.nonzero(am[b]).flatten()
            idx[b, :len(v)] = v
        idx_d = idx.to(embeds.device)
        comp = torch.gather(embeds, 1, idx_d[:, :, None].expand(-1, -1, embeds.shape[-1]))

        def restore(logits):
            out = torch.zeros_like(logits)
            for b in range(B):
                out[b, idx_d[b, :lens[b]]] = logits[b, :lens[b]]
            return out
        return comp, lens, restore

    # ------------------------------------------------------------------ generate
    @torch.no_grad()
    def generate(self, input_ids=None, images=None, regions=None, do_sample=False, temperature=1.0, top_p=None,
                 top_k=None, max_new_tokens=32, use_cache=True, stopping_criteria=None, attention_mask=None,
                 eos_token_id=None, pad_token_id=None, inputs=None, sync_every=16, num_beams=1, length_penalty=1.0,
                 early_stopping=False, num_return_sequences=1, repetition_penalty=1.0, no_repeat_ngram_size=0,
                 min_length=0, min_new_tokens=0, **kwargs):
        """Greedy (or sampled) decoding with the reference call signature
        (inference_image.py:53-61, app.py:562-571). Returns input_ids followed by the generated ids,
        like HF `generate` for decoder-only models.

        Both modes replay the same CUDA-graphed decode step; do_sample=True ends it with the device sampler
        (temperature, top_k, top_p, Philox draw) instead of the arg-max. Its seed is drawn once per call from torch's
        default CPU generator, so `torch.manual_seed(s)` makes a sampled call reproducible.

        num_beams > 1 (with do_sample=False) is HF 4.31 beam search, stated in vitron_b200.beam: length_penalty divides
        a hypothesis's summed log-probabilities by its whole length (prompt included) to that power, early_stopping is
        True, False or "never", and the best num_return_sequences hypotheses of each request are returned, request-major,
        as [B * num_return_sequences, input_len + gen_len]. The prompt (and its images) is prefilled once per request;
        its beams share its KV pages, and the beam step runs on the device inside the graphed decode step, so the host
        reads the done flags once per `sync_every` steps. With stopping_criteria the running beams are rebuilt after
        every step (beams reorder their history), which syncs once per step.

        do_sample=True with num_beams > 1 is HF 4.31 beam sampling (`beam_sample`), stated in vitron_b200.beam: the
        warpers (temperature, top_k at least 2, top_p keeping at least 2) apply to the running scores, 2 * num_beams
        candidates per search are drawn without replacement on the device, and the scorer is beam search's.
        num_return_sequences = r runs r independent searches per request and returns each one's best hypothesis:
        [B * r, input_len + gen_len], request-major; B * r * num_beams rows must fit the engine's max_batch. The seed is
        drawn from torch's default CPU generator as in sampling; prefill, page sharing, sync_every and
        stopping_criteria behave as in beam search.

        repetition_penalty, no_repeat_ngram_size, min_length and min_new_tokens are HF 4.31's logits processors, stated
        in vitron_b200.processors and enabled by 4.31's rules (repetition_penalty != 1.0, no_repeat_ngram_size > 0, and
        with an EOS id, min_length > 0 / min_new_tokens > 0; min_length counts input_ids.shape[1] + generated tokens).
        They see input_ids as 4.31 does (image and region sentinels one position each, left padding included) followed by
        the generated ids, and apply in every mode, first token included: to the logits before the arg-max or the
        sampler's warpers, and in the beam modes to the log-probabilities before the beam scores are added. They run on
        the device inside the graphed decode step. Sentinel ids are never penalised or banned (4.31 fails on them)."""
        if input_ids is None:
            input_ids = inputs
        eos = self.config.eos_token_id if eos_token_id is None else eos_token_id
        pad = self.config.pad_token_id if pad_token_id is None else pad_token_id
        eos_set = set(eos if isinstance(eos, (list, tuple)) else [eos]) if eos is not None else set()
        B = input_ids.shape[0]
        beam_search = num_beams > 1 and not do_sample
        beam_sample = num_beams > 1 and do_sample
        if beam_search:
            if num_return_sequences > num_beams:
                raise ValueError(f"num_return_sequences ({num_return_sequences}) has to be smaller or equal to "
                                 f"num_beams ({num_beams})")
            if B * num_beams > self.engine.max_batch:
                raise ValueError(f"batch {B} x num_beams {num_beams} = {B * num_beams} rows > engine max_batch "
                                 f"{self.engine.max_batch}")
        if beam_sample and B * num_return_sequences * num_beams > self.engine.max_batch:
            raise ValueError(f"batch {B} x num_return_sequences {num_return_sequences} x num_beams {num_beams} = "
                             f"{B * num_return_sequences * num_beams} rows > engine max_batch {self.engine.max_batch}")
        eos_list = sorted(eos_set) if not isinstance(eos, (list, tuple)) else [int(e) for e in eos]
        proc_settings, proc_on = processors.check_settings(repetition_penalty, no_repeat_ngram_size, min_length,
                                                           min_new_tokens, eos_list)
        self._kv_segments = None          # the prefill and decode below overwrite the cache: every handle becomes stale
        if images is not None:
            _, _, am, _, embeds, _ = self.prepare_inputs_labels_for_multimodal(
                input_ids, None, attention_mask if attention_mask is not None else torch.ones_like(input_ids),
                None, None, images, regions)
        else:
            embeds = self.model.embed_tokens(input_ids)
            am = attention_mask
        embeds, lens, _ = self._right_pad(embeds, am)
        eng = self.engine
        if proc_on:    # every engine row gets its request's raw input_ids row (a beam row its search's request)
            rows = num_beams * (num_return_sequences if beam_sample else 1) if num_beams > 1 else 1
            eng.set_processors(input_ids.detach().cpu().repeat_interleave(rows, 0), eos_ids=eos_list, **proc_settings)
        else:
            eng.clear_processors()
        logits = eng.prefill(embeds, lens)
        if do_sample:
            seed = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64)) & (2 ** 64 - 1)
            eng.set_sampling(temperature, top_k, top_p, seed)
        if beam_search or beam_sample:
            return self._beam_search(input_ids, logits, num_beams, num_return_sequences, length_penalty, early_stopping,
                                     eos_list, pad, max_new_tokens, stopping_criteria, sync_every, sample=beam_sample)
        if proc_on:
            eng.process_logits(logits)                                # generated token 0: nothing generated yet
        if do_sample:
            first = eng.sample_advance(logits)                        # generated token 0: Philox step 0
        else:
            first = ops.argmax_rows(logits)
        eng.start_decode(first, max_new_tokens)
        done_at = [None] * B  # index of the last kept token per sequence
        produced = 1
        stop_all = None
        while True:
            # examine everything produced so far (host sync once per chunk, not per token)
            toks = eng.token_log[:B, :produced].cpu()
            for b in range(B):
                if done_at[b] is None:
                    for t in range(toks.shape[1]):
                        if int(toks[b, t]) in eos_set:
                            done_at[b] = t
                            break
            if stopping_criteria is not None and stop_all is None:
                for t in range(1, produced + 1):
                    seq = torch.cat([input_ids.cpu(), self._finalize(toks[:, :t], done_at, pad)], 1)
                    if self._criteria_met(stopping_criteria, seq.to(input_ids.device)):
                        stop_all = t
                        break
            if stop_all is not None or all(d is not None for d in done_at) or produced >= max_new_tokens:
                break
            n = min(sync_every, max_new_tokens - produced)
            eng.decode_steps(B, n, sampled=do_sample)
            produced += n
        keep = produced if stop_all is None else stop_all
        if all(d is not None for d in done_at):
            keep = min(keep, max(d for d in done_at) + 1)
        toks = eng.token_log[:B, :keep].cpu()
        gen = self._finalize(toks, done_at, pad)
        return torch.cat([input_ids, gen.to(input_ids.device)], 1)

    def _beam_search(self, input_ids, logits, k, nrs, length_penalty, early_stopping, eos, pad, max_new_tokens,
                     stopping_criteria, sync_every, sample=False):
        eng = self.engine
        n_in = input_ids.shape[1]
        # beam sampling runs nrs searches per request and keeps the best of each; beam search keeps nrs of one search
        searches, keep = (nrs, 1) if sample else (1, nrs)
        prompts = input_ids.repeat_interleave(searches, 0)   # the prompt of each search
        B = prompts.shape[0]
        R = B * k
        if pad is None:
            pad = eos[0] if eos else 0
        prm = dict(length_penalty=float(length_penalty), early_stopping=early_stopping, pad=int(pad), input_len=n_in,
                   max_length=n_in + max_new_tokens, eos=eos)
        eng.start_beam(logits, k, max_new_tokens, beam.pack_params(length_penalty, early_stopping, pad, n_in,
                                                                   n_in + max_new_tokens, eos),
                       sample=sample, searches=searches)
        st = eng.beam
        produced = 1
        while produced < max_new_tokens:
            if bool(st["done"][:B].cpu().all()):
                break
            if stopping_criteria is not None:
                seq = torch.cat([prompts.cpu().repeat_interleave(k, 0), self._running(produced, R)], 1)
                if self._criteria_met(stopping_criteria, seq.to(input_ids.device)):
                    break
            n = 1 if stopping_criteria is not None else min(sync_every, max_new_tokens - produced)
            eng.decode_steps(R, n, sampled="beam_sample" if sample else "beam")
            produced += n
        done = st["done"][:B].cpu().tolist()
        hs, hl, hq = st["hyp_score"][:R].cpu(), st["hyp_len"][:R].cpu(), st["hyp_seq"][:R].cpu()
        counts, ids = st["hyp_count"][:B].cpu().tolist(), st["hyp_ids"][:R].cpu()
        hyps = []
        for b in range(B):
            h = beam.Hypotheses(k, prm["length_penalty"], early_stopping, prm["max_length"])
            h.slots = [dict(score=float(hs[b * k + s]), length=int(hl[b * k + s]), seq=int(hq[b * k + s]),
                            ids=ids[b * k + s, :int(hl[b * k + s]) - n_in]) for s in range(counts[b])]
            hyps.append(h)
        gen = beam.finalize(hyps, done, st["beam_score"][:R].cpu(), self._running(produced, R), keep, prm)
        return torch.cat([prompts.repeat_interleave(keep, 0), gen.to(input_ids.device)], 1)

    def _running(self, t, R):
        eng = self.engine
        return beam.running_ids(eng.beam["beam_src"][:R].cpu(), eng.token_log[:R].cpu(), eng.d_prompt[:R].cpu(), t)

    @staticmethod
    def _finalize(toks, done_at, pad):
        out = toks.clone()
        for b, d in enumerate(done_at):
            if d is not None and d + 1 < out.shape[1]:
                out[b, d + 1:] = pad
        return out

    @staticmethod
    def _criteria_met(criteria, seq):
        try:
            r = criteria(seq, None)
        except TypeError:
            r = any(c(seq, None) for c in criteria)
        if isinstance(r, torch.Tensor):
            return bool(r.all())
        return bool(r)


LlavaLlamaForCausalLM = VitronLlamaForCausalLM  # the reference's class name
