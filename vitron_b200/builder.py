"""`load_pretrained_model` with the reference's signature and return value (vitron/model/builder.py:27-171):

    tokenizer, model, {'image': image_processor, 'video': video_processor}, context_len =
        load_pretrained_model(model_path, model_base, model_name, load_8bit=False, load_4bit=False,
                              device_map="auto", device="cuda", **kwargs)

so that `inference_image.py:19` / `inference_video.py` / `app.py` run unchanged after
`from vitron_b200.builder import load_pretrained_model`. The model returned is the CUDA drop-in
(`VitronLlamaForCausalLM`), the processors are the device-side LanguageBind transforms.

What the reference's loader does through `transformers` / `peft`, restated on plain files (neither library is needed to
read a checkpoint directory):
  * merged checkpoint (`model_base is None`): `config.json` + `pytorch_model*.bin` / `*.safetensors` shards (builder.py:104-110);
  * LoRA checkpoint (`'lora' in model_name`, builder.py:52-84): base weights from `model_base`, `non_lora_trainables.bin` with the
    reference's key-prefix stripping (:76-79), then `adapter_model.{bin,safetensors}` merged as
    W += (lora_B @ lora_A) * lora_alpha / r  — the arithmetic of `PeftModel.merge_and_unload()` (:83-84);
  * projector-only checkpoint (`model_base` given, no 'lora', builder.py:85-103): base weights + `mm_projector.bin`;
  * special tokens added to the tokenizer and the embeddings resized (builder.py:139-146);
  * 4-bit loading (`load_4bit=True`, bitsandbytes NF4 with double-quantised scales, :36-46): the language model's
    projections, the mm_projector and the region extractor are quantised with vitron_b200.nf4 and served by the NF4
    kernels; embed_tokens, lm_head and the vision towers stay bf16. A LoRA is merged in float BEFORE quantisation (the
    reference runs it through peft on the quantised base instead);
  * 8-bit loading (LLM.int8, whose outlier decomposition depends on the activations) is not offered: a request raises
    ValueError.
`cache_dir`, `device_map`, `torch_dtype` keywords are accepted and ignored like any other `from_pretrained` keyword the
CUDA path has no use for. Extra keywords: `tokenizer=` (a ready tokenizer object instead of `AutoTokenizer.from_pretrained`),
`max_batch=` / `max_seq_len=` (KV-cache capacity of the engine; default 8 x context_len)."""
import glob
import json
import os
import warnings

import torch

from .processing import LanguageBindImageProcessor, LanguageBindVideoProcessor
from .vision_tower import VisionConfig
from .vitron_model import VitronConfig, VitronLlamaForCausalLM

# vitron/constants.py
DEFAULT_IMAGE_PATCH_TOKEN, DEFAULT_VIDEO_PATCH_TOKEN = "<im_patch>", "<vid_patch>"
DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN = "<im_start>", "<im_end>"
DEFAULT_VID_START_TOKEN, DEFAULT_VID_END_TOKEN = "<vid_start>", "<vid_end>"

LANGUAGEBIND_VIT_L14 = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                            image_size=224, patch_size=14, hidden_act="gelu", layer_norm_eps=1e-5)


def _read_json(path):
    with open(path) as f:
        return json.load(f)


def _load_file(path):
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path, device="cpu")
    return torch.load(path, map_location="cpu", weights_only=True)


def load_checkpoint_dir(path):
    """name -> CPU tensor of every weight shard in a HF-style directory (index json, *.safetensors or pytorch_model*.bin)."""
    for idx in ("model.safetensors.index.json", "pytorch_model.bin.index.json"):
        ip = os.path.join(path, idx)
        if os.path.exists(ip):
            files = sorted(set(_read_json(ip)["weight_map"].values()))
            break
    else:
        files = sorted(os.path.basename(f) for f in glob.glob(os.path.join(path, "*.safetensors")) if "adapter" not in os.path.basename(f))
        if not files:
            files = sorted(os.path.basename(f) for f in glob.glob(os.path.join(path, "pytorch_model*.bin")))
    if not files:
        raise FileNotFoundError(f"no weight shards (*.safetensors / pytorch_model*.bin) under {path}")
    sd = {}
    for f in files:
        sd.update(_load_file(os.path.join(path, f)))
    return sd


def merge_lora(sd, adapter_sd, adapter_cfg):
    """`PeftModel.merge_and_unload()` for plain Linear LoRA adapters: W += (B @ A) * (lora_alpha / r), in fp32."""
    scale = float(adapter_cfg.get("lora_alpha", 1)) / float(adapter_cfg.get("r", 1))
    pairs = {}
    for k, v in adapter_sd.items():
        for tag in (".lora_A.", ".lora_B."):
            if tag in k:
                base = k.split(tag)[0]
                for pre in ("base_model.model.", "base_model."):
                    if base.startswith(pre):
                        base = base[len(pre):]
                        break
                pairs.setdefault(base, {})[tag[6]] = v
    merged = 0
    for base, ab in pairs.items():
        name = base + ".weight"
        if name not in sd:
            alt = name[6:] if name.startswith("model.") and name[6:] in sd else None
            if alt is None:
                raise KeyError(f"LoRA adapter targets {name}, which the base checkpoint does not hold")
            name = alt
        if "A" not in ab or "B" not in ab:
            raise KeyError(f"incomplete LoRA pair for {base}")
        w = sd[name].float() + (ab["B"].float() @ ab["A"].float()) * scale
        sd[name] = w.to(sd[name].dtype)
        merged += 1
    return merged


def _vision_cfg(cfg, key, cache_dir, video):
    """VisionConfig of the tower named by config[key]: its own config.json when the tower directory is on disk (the
    `vision_config` block of the LanguageBind checkpoints), else the LanguageBind ViT-L/14 values (SURVEY.md §8)."""
    name = cfg.get(key)
    if name is None:
        return None
    v = dict(LANGUAGEBIND_VIT_L14)
    for root in (name, os.path.join(cache_dir or "", name), os.path.join(cache_dir or "", os.path.basename(str(name)))):
        cj = os.path.join(str(root), "config.json")
        if os.path.exists(cj):
            vc = _read_json(cj)
            vc = vc.get("vision_config", vc)
            v.update({k: vc[k] for k in ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "image_size",
                                         "patch_size", "hidden_act", "layer_norm_eps", "num_frames") if k in vc})
            break
    if video:
        v.update(add_time_attn=True, num_frames=int(v.get("num_frames", cfg.get("num_frames", 8))))
    else:
        v.pop("num_frames", None)
    return VisionConfig(**v)


def load_pretrained_model(model_path, model_base, model_name, load_8bit=False, load_4bit=False, device_map="auto", device="cuda",
                          **kwargs):
    if load_8bit:
        raise ValueError("vitron_b200 does not offer 8-bit loading (LLM.int8, builder.py:36-39); load_4bit=True serves NF4")
    cache_dir = kwargs.pop("cache_dir", None)
    tokenizer = kwargs.pop("tokenizer", None)
    max_batch = int(kwargs.pop("max_batch", 8))
    dev = torch.device(device if device != "cuda" else f"cuda:{torch.cuda.current_device()}" if torch.cuda.is_available() else device)
    name = model_name.lower()
    is_llava = "llava" in name
    if "mpt" in name:
        raise ValueError("the MPT language model (builder.py:88-93) is outside this path (SURVEY.md §2)")
    if is_llava and "lora" in name and model_base is None:
        warnings.warn("There is `lora` in model name but no `model_base` is provided.")  # builder.py:50-51
    cfg_dir = model_path
    weights_dir = model_base if model_base is not None else model_path
    cfg = _read_json(os.path.join(cfg_dir, "config.json"))
    if tokenizer is None:
        from transformers import AutoTokenizer
        tokenizer = AutoTokenizer.from_pretrained(weights_dir if model_base is not None else model_path, use_fast=False)

    sd = load_checkpoint_dir(weights_dir)
    if model_base is not None and is_llava and "lora" in name:
        nl = os.path.join(model_path, "non_lora_trainables.bin")
        if os.path.exists(nl):
            extra = _load_file(nl)
            extra = {(k[11:] if k.startswith("base_model.") else k): v for k, v in extra.items()}       # builder.py:76
            if any(k.startswith("model.model.") for k in extra):
                extra = {(k[6:] if k.startswith("model.") else k): v for k, v in extra.items()}             # builder.py:77-78
            sd.update(extra)
        for an in ("adapter_model.safetensors", "adapter_model.bin"):
            ap = os.path.join(model_path, an)
            if os.path.exists(ap):
                merge_lora(sd, _load_file(ap), _read_json(os.path.join(model_path, "adapter_config.json")))
                break
    elif model_base is not None and is_llava:
        sd.update({k: v for k, v in _load_file(os.path.join(model_path, "mm_projector.bin")).items()})        # builder.py:101-103

    context_len = int(cfg.get("max_sequence_length", 2048))                                                    # builder.py:166-169
    llm = {k: cfg[k] for k in ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "vocab_size",
                               "rms_norm_eps", "rope_theta", "max_position_embeddings") if k in cfg}
    if "lm_head.weight" in sd:
        llm["vocab_size"] = sd["lm_head.weight"].shape[0]
    vcfg = VitronConfig(llm=llm, vision=_vision_cfg(cfg, "mm_image_tower", cache_dir, False) if is_llava else None,
                        video=_vision_cfg(cfg, "mm_video_tower", cache_dir, True) if is_llava else None,
                        mm_projector_type=cfg.get("mm_projector_type", "linear"),
                        mm_vision_select_layer=cfg.get("mm_vision_select_layer", -2),
                        mm_vision_select_feature=cfg.get("mm_vision_select_feature", "patch"),
                        tokenizer_padding_side=getattr(tokenizer, "padding_side", "right"),
                        tokenizer_model_max_length=getattr(tokenizer, "model_max_length", None),
                        pad_token_id=cfg.get("pad_token_id", 0), eos_token_id=cfg.get("eos_token_id", 2),
                        bos_token_id=cfg.get("bos_token_id", 1), mm_image_tower=cfg.get("mm_image_tower"),
                        mm_video_tower=cfg.get("mm_video_tower"), mm_use_im_start_end=cfg.get("mm_use_im_start_end", False),
                        mm_use_im_patch_token=cfg.get("mm_use_im_patch_token", True), max_sequence_length=context_len)
    model = VitronLlamaForCausalLM(vcfg, dev, max_batch=max_batch, max_seq_len=int(kwargs.pop("max_seq_len", context_len)))
    # towers whose weights are not inside the checkpoint are left unloaded exactly like `is_loaded == False` in the reference
    model.load_state_dict(sd, nf4=bool(load_4bit))
    del sd

    processor = {"image": None, "video": None}
    if is_llava:
        if vcfg.mm_use_im_patch_token:                                                                           # builder.py:139-142
            tokenizer.add_tokens([DEFAULT_IMAGE_PATCH_TOKEN], special_tokens=True)
            tokenizer.add_tokens([DEFAULT_VIDEO_PATCH_TOKEN], special_tokens=True)
        if vcfg.mm_use_im_start_end:
            tokenizer.add_tokens([DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN], special_tokens=True)
            tokenizer.add_tokens([DEFAULT_VID_START_TOKEN, DEFAULT_VID_END_TOKEN], special_tokens=True)
        model.resize_token_embeddings(len(tokenizer))
        if vcfg.mm_image_tower is not None:
            tower = model.get_image_tower()
            tower.to(device=dev, dtype=torch.float16)      # builder.py:153 (accepted, served in bf16)
            tower.image_processor = LanguageBindImageProcessor(device=dev, dtype=torch.bfloat16)
            processor["image"] = tower.image_processor
        if vcfg.mm_video_tower is not None:
            tower = model.get_video_tower()
            tower.to(device=dev, dtype=torch.float16)
            tower.video_processor = LanguageBindVideoProcessor(device=dev, dtype=torch.bfloat16)
            processor["video"] = tower.video_processor
    return tokenizer, model, processor, context_len
