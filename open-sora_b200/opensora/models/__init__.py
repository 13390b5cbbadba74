from . import hunyuan_vae, mmdit, stdit, text, text_encoder  # noqa: F401  (registers "hunyuan_vae", "STDiT3-XL/2", "text_embedder", "t5", ... in opensora.registry.MODELS)
