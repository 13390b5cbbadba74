from . import conditioner  # noqa: F401  (registers "text_embedder" in opensora.registry.MODELS)
