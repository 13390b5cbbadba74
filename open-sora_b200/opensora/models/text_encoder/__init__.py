from .t5 import T5Encoder  # noqa: F401  (registers "t5" in opensora.registry.MODELS)
