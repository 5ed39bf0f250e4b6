"""vitron_b200 — H100-native (sm_90a) kernels behind SkyworkAI/Vitron's multimodal forward path.

Public drop-in surface (reference names): VitronLlamaForCausalLM / LlavaLlamaForCausalLM,
LanguageBindImageTower / LanguageBindVideoTower, build_vision_projector, build_region_extractor,
RegionExtractor, UNetSD_I2VGen, GatedSelfAttentionDense, SEEM decoders — see DESIGN.md.
Importing the package does not load the CUDA library; the first op does (and raises if missing).
"""
__version__ = "0.1.0"
