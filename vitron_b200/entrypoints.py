"""The module-level entry points of the reference's `modules/*` with their own signatures (SURVEY.md §8b face 1), as thin
orchestration over the CUDA pipelines of this package:

  reference                                                                 here
  ------------------------------------------------------------------------  --------------------------------------------
  modules/GLIGEN/demo/gligen/task_grounded_generation.py:185                grounded_generation_box(loaded_model_list, instruction, *args, **kwargs)
  modules/GLIGEN/demo/gligen/task_grounded_generation.py:66                 load_ckpt(config, state_dict)
  modules/GLIGEN/demo/app.py:270                                            generate(task, language_instruction, grounding_texts, sketch_pad, ...)
  modules/SEEM/demo_code/app.py:79                                          inference(image, task, *args, **kwargs)
  modules/i2vgen-xl/tools/inferences/inference_i2vgen_entrance.py:36        inference_i2vgen_entrance(cfg_update, **kwargs)
  app.py:316                                                                image_to_video(image_path=None, text_prompt=None)

What stays outside (host-only, no arithmetic of the path): PIL / gradio widgets, file I/O of results, the CLIP BPE / sentencepiece
vocabularies (not in the tree: checkpoints/README.md:15). Those are INJECTED: every function takes the objects the reference builds
in its module globals (`model`, `pipe`, `clip_model` ...) through `configure(...)` or keyword arguments, and fails with a clear
error when one is missing — never with a silent CPU fallback. Tensors in, tensors out; the reference's PIL conversions are one
`numpy()` call on the returned tensors."""
import json
import random
from functools import partial

import numpy as np
import torch

_STATE = {}


def configure(**objects):
    """Register the long-lived objects the reference keeps in module globals: `seem_model` (callable features -> outputs),
    `seem_backbone`, `gligen_models` (model, autoencoder, text_encoder, diffusion), `gligen_clip` (dict of feature callables),
    `i2vgen_pipeline` (vitron_b200.i2vgen_pipeline.I2VGenXLPipeline), `i2vgen_tokenize`, `load_image`, `save_video`."""
    _STATE.update(objects)
    return _STATE


def _need(name, hint):
    if name not in _STATE or _STATE[name] is None:
        raise RuntimeError(f"vitron_b200.entrypoints: `{name}` is not configured ({hint}); call entrypoints.configure({name}=...)")
    return _STATE[name]


# =========================================================================================== GLIGEN
def complete_mask(has_mask, max_objs):
    """task_grounded_generation.py:139-147."""
    mask = torch.ones(1, max_objs)
    if type(has_mask) == int or type(has_mask) == float:
        return mask * has_mask
    for idx, value in enumerate(has_mask):
        mask[0, idx] = value
    return mask


def prepare_grounding_batch(meta, batch=1, max_objs=30, clip_model=None, device="cuda", embed_dim=768):
    """`fire_clip` (task_grounded_generation.py:150-182) with the CLIP feature extraction injected: `clip_model` is a dict
    with callables `text_feature(phrase) -> [1, 768]` (pooler output before projection) and `image_feature(image) -> [1, 768]`
    (re-projected, renormalised x 28.7) — the two branches of `get_clip_feature` (:105-136)."""
    phrases, images = meta["phrases"], meta["images"]
    boxes = torch.zeros(max_objs, 4)
    masks = torch.zeros(max_objs)
    text_embeddings = torch.zeros(max_objs, embed_dim)     # 768 = CLIP ViT-L/14 (the reference hard-codes it, :165-166)
    image_embeddings = torch.zeros(max_objs, embed_dim)
    if len(phrases) > 0:
        if clip_model is None:
            raise RuntimeError("grounding phrases / images given but no clip_model={'text_feature':..., 'image_feature':...}")
        tf = torch.cat([clip_model["text_feature"](p).float().cpu().reshape(1, -1) if p is not None else torch.zeros(1, embed_dim)
                        for p in phrases], 0)
        imf = torch.cat([clip_model["image_feature"](im).float().cpu().reshape(1, -1) if im is not None else torch.zeros(1, embed_dim)
                         for im in images], 0)
        for idx, (box, t, i) in enumerate(zip(meta["locations"], tf, imf)):
            boxes[idx] = torch.tensor(box)
            masks[idx] = 1
            text_embeddings[idx] = t
            image_embeddings[idx] = i
    out = {"boxes": boxes.unsqueeze(0).repeat(batch, 1, 1), "masks": masks.unsqueeze(0).repeat(batch, 1),
           "text_masks": masks.unsqueeze(0).repeat(batch, 1) * complete_mask(meta["has_text_mask"], max_objs),
           "image_masks": masks.unsqueeze(0).repeat(batch, 1) * complete_mask(meta["has_image_mask"], max_objs),
           "text_embeddings": text_embeddings.unsqueeze(0).repeat(batch, 1, 1),
           "image_embeddings": image_embeddings.unsqueeze(0).repeat(batch, 1, 1)}
    return {k: v.to(device) for k, v in out.items()}


def draw_masks_from_boxes(boxes, size):
    """gligen/ldm/util.py draw_masks_from_boxes: 1 outside the boxes, 0 inside (the region to inpaint)."""
    h, w = (size, size) if isinstance(size, int) else size
    image_masks = []
    for box_set in boxes:
        m = torch.ones(h, w)
        for box in box_set if isinstance(box_set[0], (list, tuple)) else [box_set]:
            x0, x1 = box[0] * w, box[2] * w
            y0, y1 = box[1] * h, box[3] * h
            m[int(y0):int(y1), int(x0):int(x1)] = 0
        image_masks.append(m)
    return torch.stack(image_masks).unsqueeze(1)


def load_ckpt(config, state_dict, device="cuda"):
    """task_grounded_generation.py:66-81 on the CUDA modules: `config` provides `model` (UNetModel kwargs), `autoencoder`
    (ddconfig, embed_dim, scale_factor), `alpha_scale`; `state_dict` the four sub-dicts. The text encoder (CLIP text
    transformer) is third-party and injected as `config['text_encoder']` (object with `.encode(list[str])`)."""
    from .autoencoder import AutoencoderKL
    from .gligen_sampler import DDPM, GligenAutoencoder, set_alpha_scale
    from .gligen_unet import UNetModel
    model = UNetModel(**config["model"], device=device).load_state_dict(state_dict["model"])
    ae = config["autoencoder"]
    vae = AutoencoderKL(ae["ddconfig"], ae.get("embed_dim", 4), device=device).load_state_dict(state_dict["autoencoder"])
    autoencoder = GligenAutoencoder(vae, ae.get("scale_factor", 0.18215))
    diffusion = DDPM(device=device, **config.get("diffusion", {}))
    set_alpha_scale(model, config.get("alpha_scale", 1.0))
    return model, autoencoder, config.get("text_encoder"), diffusion


@torch.no_grad()
def grounded_generation_box(loaded_model_list, instruction, *args, **kwargs):
    """task_grounded_generation.py:185-298 up to the decoded samples: returns (sample_list, overlay_list) where each sample is a
    uint8 HWC tensor (the reference's `Image.fromarray` input) and overlay_list the normalised boxes to draw."""
    from .gligen_sampler import GligenAutoencoder, PLMSSampler, alpha_generator, set_alpha_scale
    model, autoencoder, text_encoder, diffusion = loaded_model_list
    if text_encoder is None:
        raise RuntimeError("loaded_model_list[2] (text_encoder with .encode(list[str])) is required")
    if not isinstance(autoencoder, GligenAutoencoder):
        autoencoder = GligenAutoencoder(autoencoder, kwargs.get("scale_factor", 0.18215))
    device = model.device
    batch_size = instruction["batch_size"]
    is_inpaint = "input_image" in instruction
    if instruction.get("fix_seed", False):                                                  # :194-198
        random_seed = instruction["rand_seed"]
        random.seed(random_seed)
        np.random.seed(random_seed)
        torch.manual_seed(random_seed)
    batch = prepare_grounding_batch(instruction, batch_size, clip_model=kwargs.get("clip_model", None), device=device,
                                    embed_dim=getattr(model, "positive_len", 768))
    context = text_encoder.encode([instruction["prompt"]] * batch_size)
    uc = text_encoder.encode(batch_size * [""])
    input = dict(x=None, timesteps=None, context=context, boxes=batch["boxes"], masks=batch["masks"],
                 text_masks=batch["text_masks"], image_masks=batch["image_masks"], text_embeddings=batch["text_embeddings"],
                 image_embeddings=batch["image_embeddings"])
    inpainting_mask = x0 = None
    if is_inpaint:                                                                           # :217-241
        img = instruction["input_image"]
        img = img if torch.is_tensor(img) else torch.from_numpy(np.asarray(img)).permute(2, 0, 1)
        input_image = (img.float().unsqueeze(0).to(device) / 255 - 0.5) / 0.5
        x0 = autoencoder.encode(input_image)
        if instruction.get("actual_mask") is not None:
            inpainting_mask = instruction["actual_mask"][None, None].expand(batch["boxes"].shape[0], -1, -1, -1).to(device)
        else:
            actual_boxes = [instruction["inpainting_boxes_nodrop"] for _ in range(batch["boxes"].shape[0])]
            inpainting_mask = draw_masks_from_boxes(actual_boxes, (x0.shape[-2], x0.shape[-1])).to(device)
        masked_x0 = x0 * inpainting_mask
        input["inpainting_extra_input"] = torch.cat([masked_x0, inpainting_mask], dim=1)
    sampler = PLMSSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=instruction["alpha_type"]),
                          set_alpha_scale=set_alpha_scale)
    steps = kwargs.get("steps", 50)
    shape = (batch_size, model.in_channels, model.image_size, model.image_size)
    if is_inpaint:
        uc = context                                                                          # :257-258
    samples_fake = sampler.sample(S=steps, shape=shape, input=input, uc=uc, guidance_scale=instruction["guidance_scale"],
                                  mask=inpainting_mask, x0=x0)
    samples_fake = autoencoder.decode(samples_fake)
    sample_list, overlay_list = [], []
    for sample in samples_fake:                                                              # :276-295 without the file writes
        sample = torch.clamp(sample.float(), min=-1, max=1) * 0.5 + 0.5
        sample_list.append((sample.permute(1, 2, 0) * 255).to(torch.uint8).cpu())
        overlay_list.append(list(instruction.get("locations", [])))
    return sample_list, overlay_list


def generate(task, language_instruction, grounding_texts, sketch_pad, alpha_sample, guidance_scale, batch_size, fix_seed, rand_seed,
             use_actual_mask, append_grounding, style_cond_image, state, inpainting_image=None, inpainting_mask=None):
    """modules/GLIGEN/demo/app.py:270-414: validates the widget state, builds the `instruction` dict and calls
    `grounded_generation_box`. Raises ValueError where the reference raises `gr.Error`."""
    if "boxes" not in state:
        state["boxes"] = []
    boxes = state["boxes"]
    if len(grounding_texts) != 0:
        grounding_texts = [x.strip() for x in grounding_texts.split(";")]
    if len(boxes) != len(grounding_texts):
        raise ValueError("There is a mismatching between bounding boxes and the given grounding instruction. Hit clear to start over.")
    if task == "Grounded Inpainting" and len(grounding_texts) == 0:
        raise ValueError("There is nothing to inpaint. Please give grounding instructions and draw the bounding box. Hit clear to start over.")
    if task == "Grounded Generation" and len(language_instruction) == 0:
        raise ValueError("There is nothing to generate. Please give language instructions. Hit clear to start over.")
    boxes = (np.asarray(boxes) / 512).tolist()
    grounding_instruction = json.dumps({obj: box for obj, box in zip(grounding_texts, boxes)})
    if append_grounding:                                                                      # auto_append_grounding :262-267
        for g in grounding_texts:
            if g not in language_instruction and g != "auto":
                language_instruction += "; " + g
    gi = json.loads(grounding_instruction)
    phrase_list, location_list = list(gi.keys()), list(gi.values())
    instruction = dict(prompt=language_instruction, phrases=phrase_list, images=[None] * len(phrase_list), locations=location_list,
                       alpha_type=[alpha_sample, 0, 1.0 - alpha_sample], has_text_mask=1, has_image_mask=0,
                       guidance_scale=guidance_scale, batch_size=batch_size, fix_seed=bool(fix_seed), rand_seed=int(rand_seed),
                       actual_mask=None, inpainting_boxes_nodrop=location_list, save_folder_name="gligen")
    if task == "Grounded Inpainting":
        image = inpainting_image if inpainting_image is not None else state.get("original_image", sketch_pad["image"] if sketch_pad else None)
        if image is None:
            raise ValueError("Grounded Inpainting needs an image")
        instruction["input_image"] = image
        if use_actual_mask:
            m = inpainting_mask if inpainting_mask is not None else sketch_pad["mask"]
            m = torch.as_tensor(np.asarray(m)).float()
            m = m[..., 0] if m.ndim == 3 else m
            instruction["actual_mask"] = 1.0 - (m > 0).float() if m.max() > 1 else 1.0 - m
    models = _need("gligen_models", "the (model, autoencoder, text_encoder, diffusion) tuple of load_ckpt")
    return grounded_generation_box(models, instruction, clip_model=_STATE.get("gligen_clip"))


# =========================================================================================== SEEM
@torch.no_grad()
def inference(image, task, *args, **kwargs):
    """modules/SEEM/demo_code/app.py:79-87 -> tasks/interactive.py:35: `image` is the widget dict {'image': HWC uint8, 'mask': ...}
    (already resized: the reference's PIL Resize(512, BICUBIC) is host-side), `task` the list of task names. Implemented: the
    prompt-free branch (`[]` / `['Panoptic']`) and the 'Stroke' (spatial), 'Text' (grounding) and 'Audio' prompts of
    seem.py:398-500 through `extra` (the text / audio encoders are injected: their towers are outside §8). Returns the
    predictor's output dict (pred_logits, pred_masks, pred_captions, pred_pspatials ...); the reference's visualiser
    (detectron2) is out of scope."""
    tasks = list(task) if task is not None else []
    unsupported = [t for t in tasks if t not in ("Panoptic", "Stroke", "Text", "Audio")]
    if unsupported:
        raise NotImplementedError(f"SEEM task(s) {unsupported}: 'Example' (reference image) goes through predictor(task='refimg') "
                                  "directly; video tracking is host-side glue over the same head")
    head = _need("seem_model", "XDecoderHead (pixel decoder + mask decoder)")
    backbone = _need("seem_backbone", "D2FocalNet backbone")
    img = image["image"] if isinstance(image, dict) else image
    img = img if torch.is_tensor(img) else torch.from_numpy(np.asarray(img))
    dev = head.predictor.device if hasattr(head, "predictor") else torch.device("cuda")
    pix = img.permute(2, 0, 1)[None].float().to(dev)
    mean = torch.tensor([123.675, 116.280, 103.530], device=pix.device).view(1, 3, 1, 1)   # seem_focall_lang.yaml INPUT.PIXEL_MEAN/STD
    std = torch.tensor([58.395, 57.120, 57.375], device=pix.device).view(1, 3, 1, 1)
    feats = backbone((pix - mean) / std)
    extra = {}
    if "Stroke" in tasks:                                       # interactive.py:96-104: the sketch mask is the positive prompt
        m = image["mask"]
        m = m if torch.is_tensor(m) else torch.from_numpy(np.asarray(m))
        m = (m[..., 0] if m.ndim == 3 else m)[None, None].float()
        m = torch.nn.functional.interpolate(m, (pix.shape[2], pix.shape[3]), mode="bilinear") > 0
        extra["spatial_query_pos_mask"] = [m[0].to(dev)]
        extra["spatial_query_neg_mask"] = [torch.zeros_like(m[0]).to(dev)]
    if "Text" in tasks:                                         # interactive.py:106-114: grounding tokens from the language encoder
        enc = _need("seem_text_encoder", "callable(list[str]) -> (tokens [T, 1, C], nonzero_mask [1, T]) of the SEEM language encoder")
        tok, nz = enc([kwargs.get("reftxt") if "reftxt" in kwargs else (args[1] if len(args) > 1 else "")])
        extra["grounding_tokens"], extra["grounding_nonzero_mask"] = tok, nz
    if "Audio" in tasks:
        enc = _need("seem_audio_encoder", "callable(audio path) -> (tokens [T, 1, C], nonzero_mask [1, T]) (whisper + language encoder)")
        tok, nz = enc(kwargs.get("audio_pth") if "audio_pth" in kwargs else (args[2] if len(args) > 2 else None))
        extra["audio_tokens"], extra["audio_nonzero_mask"] = tok, nz
    return head(feats, extra=extra)


# =========================================================================================== i2vgen-xl
@torch.no_grad()
def inference_i2vgen_entrance(cfg_update, **kwargs):
    """modules/i2vgen-xl/tools/inferences/inference_i2vgen_entrance.py:36 -> worker :59-209 for ONE process: for every
    `image_path|||caption` line of cfg_update['test_list_path'] (or cfg_update['test_list']) run the configured
    I2VGenXLPipeline and hand the video tensor to `save_video(name, video)`. The YAML config system, logging and the
    torch.multiprocessing spawn of the reference are host plumbing and not reproduced: `cfg_update` is read as a plain dict."""
    pipe = _need("i2vgen_pipeline", "vitron_b200.i2vgen_pipeline.I2VGenXLPipeline")
    tokenize = _need("i2vgen_tokenize", "open_clip tokenizer: str -> [1, 77] ids")
    load_image = _need("load_image", "path -> (image_vit [1,3,224,224], image_vae [1,3,H,W]) after the reference's transforms")
    save_video = _STATE.get("save_video")
    cfg = dict(cfg_update)
    cfg.update(kwargs)
    lines = cfg.get("test_list")
    if lines is None:
        with open(cfg["test_list_path"]) as f:
            lines = [ln.strip() for ln in f.readlines()]
    neg = cfg.get("negative_prompt", "Distorted, discontinuous, Ugly, blurry, low resolution, motionless, static, disfigured, "
                                     "disconnected limbs, Ugly faces, incomplete arms")
    out = []
    for _ in range(int(cfg.get("round", 1))):
        for line in lines:
            if line.startswith("#"):
                continue
            img_key, caption = line.split("|||")
            if caption == "":
                continue
            image_vit, image_vae = load_image(img_key)
            video = pipe(image_vit, image_vae, tokenize(caption), tokenize(neg), generator=cfg.get("generator"))
            out.append((img_key, video))
            if save_video is not None:
                save_video(img_key, video)
    return out


def image_to_video(image_path=None, text_prompt=None):
    """app.py:316-343 (the diffusers `I2VGenXLPipeline` route of the Gradio app): same contract on the UNetSD_I2VGen pipeline —
    returns what `save_video` returns (a path) or the video tensor when no saver is configured."""
    if image_path is None or text_prompt is None:
        return None, None
    pipe = _need("i2vgen_pipeline", "vitron_b200.i2vgen_pipeline.I2VGenXLPipeline")
    tokenize = _need("i2vgen_tokenize", "open_clip tokenizer: str -> [1, 77] ids")
    load_image = _need("load_image", "path -> (image_vit, image_vae)")
    negative_prompt = "Distorted, discontinuous, Ugly, blurry, low resolution, motionless, static, disfigured, disconnected limbs, Ugly faces, incomplete arms"
    generator = torch.Generator().manual_seed(8800)
    image_vit, image_vae = load_image(image_path)
    video = pipe(image_vit, image_vae, tokenize(text_prompt), tokenize(negative_prompt), generator=generator)
    saver = _STATE.get("save_video")
    return saver(image_path, video) if saver is not None else video
