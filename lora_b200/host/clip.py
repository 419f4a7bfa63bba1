"""Text encoder host models: transformers' CLIPTextModel, random-initialised (no weights offline).

SD1.5: CLIP ViT-L/14 text (768 wide, 12 layers, 12 heads, quick_gelu). The reference injects LoRA
into its `CLIPAttention` blocks (lora_diffusion/lora.py:163; train_lora_dreambooth.py:608-613): 12
layers x {k_proj, v_proj, q_proj, out_proj} = 48 sites of (77, 768 -> 768).
SD 2.x: OpenCLIP ViT-H/14 text as diffusers ships it (1024 wide, 23 layers, 16 heads, gelu): 92
sites of (77, 1024 -> 1024).
SDXL: the ViT-L encoder above plus OpenCLIP ViT-bigG/14 text as diffusers ships it in `text_encoder_2`
(a CLIPTextModelWithProjection: 1280 wide, 32 layers, 20 heads, gelu, text_projection 1280 -> 1280):
48 + 128 sites, the second set of (77, 1280 -> 1280)."""
from transformers import CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection


def sd15_text_config(tiny: bool = False) -> CLIPTextConfig:
    if tiny:
        return CLIPTextConfig(vocab_size=1000, hidden_size=48, intermediate_size=96,
                              num_hidden_layers=2, num_attention_heads=2,
                              max_position_embeddings=77, hidden_act="quick_gelu",
                              projection_dim=48)
    return CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072,
                          num_hidden_layers=12, num_attention_heads=12,
                          max_position_embeddings=77, hidden_act="quick_gelu",
                          projection_dim=768)


def sd2_text_config(tiny: bool = False) -> CLIPTextConfig:
    if tiny:       # width 64 != the tiny SD2 UNet's 32: cross-attention K differs from the UNet's
        return CLIPTextConfig(vocab_size=1000, hidden_size=64, intermediate_size=128,
                              num_hidden_layers=2, num_attention_heads=4,
                              max_position_embeddings=77, hidden_act="gelu",
                              projection_dim=64)
    return CLIPTextConfig(vocab_size=49408, hidden_size=1024, intermediate_size=4096,
                          num_hidden_layers=23, num_attention_heads=16,
                          max_position_embeddings=77, hidden_act="gelu",
                          projection_dim=512)


def build_text_encoder(tiny: bool = False, sd2: bool = False) -> CLIPTextModel:
    """sd2=False: the SD1.5 encoder; sd2=True: the SD 2.x one (pair with UNetConfig.sd21 / sd2_tiny)."""
    cfg = sd2_text_config(tiny) if sd2 else sd15_text_config(tiny)
    cfg._attn_implementation = "sdpa"
    return CLIPTextModel(cfg)


def sdxl_text_config_2(tiny: bool = False) -> CLIPTextConfig:
    """SDXL's second encoder. The tiny one is 40 wide (the tiny ViT-L one is 48): the concatenated context
    (88) is wider than either. Its bos / eos ids lie inside the tiny vocabulary, so the pooled token is
    the first eos of the prompt, as with the real tokenizer."""
    if tiny:
        return CLIPTextConfig(vocab_size=1000, hidden_size=40, intermediate_size=80,
                              num_hidden_layers=2, num_attention_heads=2,
                              max_position_embeddings=77, hidden_act="gelu",
                              projection_dim=40, bos_token_id=998, eos_token_id=999)
    return CLIPTextConfig(vocab_size=49408, hidden_size=1280, intermediate_size=5120,
                          num_hidden_layers=32, num_attention_heads=20,
                          max_position_embeddings=77, hidden_act="gelu",
                          projection_dim=1280)


def build_sdxl_text_encoders(tiny: bool = False):
    """(text_encoder, text_encoder_2) of SDXL: the SD1.5 CLIPTextModel and a CLIPTextModelWithProjection
    (pair with UNetConfig.sdxl / sdxl_tiny). The tiny first encoder is host/clip.py's tiny SD1.5 one with
    the second's in-vocabulary eos id."""
    cfg1 = sd15_text_config(tiny)
    if tiny:
        cfg1.bos_token_id, cfg1.eos_token_id = 998, 999
    cfg2 = sdxl_text_config_2(tiny)
    cfg1._attn_implementation = cfg2._attn_implementation = "sdpa"
    return CLIPTextModel(cfg1), CLIPTextModelWithProjection(cfg2)
