"""VitronLlamaForCausalLM — drop-in for the reference's LlavaLlamaForCausalLM on H100 kernels.

Mirrors vitron/model/language_model/llava_llama.py:40-114 (`forward`, `generate` via HF
GenerationMixin, `prepare_inputs_for_generation`) and vitron/model/llava_arch.py:153-573
(`encode_images`, `encode_videos`, `prepare_inputs_labels_for_multimodal`) — same method names,
argument meaning, sentinel handling (IMAGE_TOKEN_INDEX -200, OBJS_TOKEN_INDEX -300), truncation and
padding rules, and the reference's parameter names for `load_state_dict`.

Mechanism: the per-sample Python cat/split loop becomes one host-side layout pass over the (tiny)
id tensor plus a single gather kernel; the decoder runs on `LlamaEngine` (paged KV cache, fused
kernels, CUDA-graph decode, arg-max on device).
"""
from types import SimpleNamespace

import torch

from . import ops
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

    def load_state_dict(self, sd, strict=True):
        """Accepts the reference's names: model.embed_tokens.*, model.layers.*, lm_head.weight,
        model.mm_projector.*, model.region_extractor.*, model.image_tower.image_tower.*,
        model.video_tower.video_tower.* (SURVEY.md Appendix B)."""
        self.engine.load_state_dict(sd)
        m = self.model
        if m.mm_projector is not None and any(k.startswith("model.mm_projector.") for k in sd):
            m.mm_projector.load_state_dict(sd, "model.mm_projector.")
        if m.region_extractor is not None and any(k.startswith("model.region_extractor.") for k in sd):
            m.region_extractor.load_state_dict(sd, "model.region_extractor.")
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
        """Full-sequence forward: logits for every position (fp32), like the reference with
        past_key_values=None. (Incremental decoding goes through `generate`, which keeps the KV cache
        inside the engine.)"""
        if past_key_values is not None:
            raise NotImplementedError("incremental forward() is internal to generate(); pass past_key_values=None")
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
        loss = None
        if labels is not None:
            sl = logits[:, :-1].reshape(-1, logits.shape[-1])
            loss = torch.nn.functional.cross_entropy(sl, labels[:, 1:].reshape(-1).to(sl.device), ignore_index=IGNORE_INDEX)
        return CausalLMOutput(loss=loss, logits=logits, past_key_values=None, hidden_states=None, attentions=None)

    __call__ = forward

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
                 eos_token_id=None, pad_token_id=None, inputs=None, sync_every=16, **kwargs):
        """Greedy (or sampled) decoding with the reference call signature
        (inference_image.py:53-61, app.py:562-571). Returns input_ids followed by the generated ids,
        like HF `generate` for decoder-only models."""
        if input_ids is None:
            input_ids = inputs
        eos = self.config.eos_token_id if eos_token_id is None else eos_token_id
        pad = self.config.pad_token_id if pad_token_id is None else pad_token_id
        eos_set = set(eos if isinstance(eos, (list, tuple)) else [eos]) if eos is not None else set()
        B = input_ids.shape[0]
        if images is not None:
            _, _, am, _, embeds, _ = self.prepare_inputs_labels_for_multimodal(
                input_ids, None, attention_mask if attention_mask is not None else torch.ones_like(input_ids),
                None, None, images, regions)
        else:
            embeds = self.model.embed_tokens(input_ids)
            am = attention_mask
        embeds, lens, _ = self._right_pad(embeds, am)
        eng = self.engine
        logits = eng.prefill(embeds, lens)
        if do_sample:
            return self._sample_loop(input_ids, logits, B, max_new_tokens, temperature, top_p, top_k, eos_set, pad,
                                     stopping_criteria)
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
            eng.decode_steps(B, n)
            produced += n
        keep = produced if stop_all is None else stop_all
        if all(d is not None for d in done_at):
            keep = min(keep, max(d for d in done_at) + 1)
        toks = eng.token_log[:B, :keep].cpu()
        gen = self._finalize(toks, done_at, pad)
        return torch.cat([input_ids, gen.to(input_ids.device)], 1)

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

    def _sample_loop(self, input_ids, logits, B, max_new_tokens, temperature, top_p, top_k, eos_set, pad, criteria):
        eng = self.engine
        out = []
        finished = torch.zeros(B, dtype=torch.bool, device=logits.device)
        for step in range(max_new_tokens):
            lg = logits.float() / max(float(temperature), 1e-6)
            if top_k:
                kth = torch.topk(lg, int(top_k), dim=-1).values[:, -1:]
                lg = lg.masked_fill(lg < kth, float("-inf"))
            if top_p is not None and top_p < 1.0:
                sl, si = torch.sort(lg, descending=True, dim=-1)
                cp = torch.softmax(sl, -1).cumsum(-1)
                rm = cp - torch.softmax(sl, -1) > top_p
                sl = sl.masked_fill(rm, float("-inf"))
                lg = torch.full_like(lg, float("-inf")).scatter(1, si, sl)
            tok = torch.multinomial(torch.softmax(lg, -1), 1).squeeze(1)
            tok = torch.where(finished, torch.full_like(tok, pad), tok)
            out.append(tok)
            for e in eos_set:
                finished |= tok == e
            seq = torch.cat([input_ids, torch.stack(out, 1).to(input_ids.device)], 1)
            if bool(finished.all()) or (criteria is not None and self._criteria_met(criteria, seq)):
                break
            if step == 0:
                eng.start_decode(tok, max_new_tokens)
            if step + 1 < max_new_tokens:
                logits = eng.decode_one_logits(tok)
        return torch.cat([input_ids, torch.stack(out, 1).to(input_ids.device)], 1)


LlavaLlamaForCausalLM = VitronLlamaForCausalLM  # the reference's class name
