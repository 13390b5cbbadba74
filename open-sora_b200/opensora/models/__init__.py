from . import hunyuan_vae, mmdit, stdit, text  # noqa: F401  (registers "hunyuan_vae", "STDiT3-XL/2", "text_embedder", ... in opensora.registry.MODELS)
