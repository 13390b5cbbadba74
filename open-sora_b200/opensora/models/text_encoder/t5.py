"""Open-Sora v1.2's text encoder for STDiT3: `T5Encoder`, registered as "t5", at v1.2's module path.  Like STDiT3 and its
sampler, v1.2's `T5Embedder` / `T5Encoder` are ABSENT from the reference tree; this is a restatement of their inference
behaviour - **parity unpinned** against v1.2's source, pinned instead against transformers' T5EncoderModel with an
attention mask (tests/golden/make_golden_t5_masked.py).

A v1.2 config names it `text_encoder = dict(type="t5", from_pretrained="DeepFloyd/t5-v1_1-xxl", model_max_length=300,
shardformer=True)`.  Prompts are tokenized to exactly `model_max_length` tokens (truncated, eos kept, right-padded) and
the tokenizer's attention mask goes into the encoder, so the pad keys are excluded in every T5 layer; the mask is also
returned for STDiT3's cross-attention.  The T5 v1.1 encoder is `text_embedder`'s (`opensora.models.text.conditioner`),
on osb200 kernels.

Precision: v1.2's inference script builds this without a dtype, i.e. T5 runs in fp32 there.  Here `dtype` may be fp32
or bf16 and the encoder always computes in bf16 (weights rounded to bf16, fp32 accumulation and softmax), so the
embeddings differ from an fp32 T5 by the bf16 noise floor of the encoder, which the tests measure.

Differences forced by the environment: there is no hub download.  `from_pretrained` is a local checkpoint directory or
a hub name already in the Hugging Face cache (`cache_dir`, else `$HF_HUB_CACHE` / `$HF_HOME/hub`), resolved as
`opensora.utils.ckpt` does; `local_files_only` is accepted and is always in effect.  Caption cleaning (v1.2's
`clean_caption`) is not done: prompts are encoded as given."""
from __future__ import annotations

import os

import torch

from opensora.models.text.conditioner import HFEmbedder
from opensora.registry import MODELS
from opensora.utils.ckpt import load_from_hf_hub

_DTYPES = (torch.float32, torch.bfloat16)


def resolve_pretrained(from_pretrained: str, cache_dir: str | None = None) -> str:
    """Local checkpoint directory of `from_pretrained`: the path itself, or the cached snapshot of a hub name."""
    if os.path.isdir(from_pretrained):
        return from_pretrained
    return os.path.dirname(load_from_hf_hub(f"{from_pretrained.rstrip('/')}/config.json", cache_dir))


@MODELS.register_module("t5")
class T5Encoder:
    """`T5Encoder(from_pretrained, model_max_length=120, device="cuda", dtype=torch.float, cache_dir=None,
    shardformer=False, local_files_only=False, tokenizer=None)`.

    `encode(text)` -> dict(y=[B, 1, L, d_model] bf16, mask=[B, L] int64) on the model's device, L = model_max_length.
    `null(n)` -> the denoiser's null caption [n, 1, L, caption_channels]; set `y_embedder = model.y_embedder` first, as
    v1.2's inference script does.  `tokenizer=` replaces the tokenizer loaded from the checkpoint directory; it must
    return `input_ids` and `attention_mask`.  `shardformer=True` changes no arithmetic (see `HFEmbedder`)."""

    def __init__(self, from_pretrained: str | None = None, model_max_length: int = 120, device="cuda",
                 dtype: torch.dtype = torch.float, cache_dir: str | None = None, shardformer: bool = False,
                 local_files_only: bool = False, tokenizer=None):
        if from_pretrained is None:
            raise ValueError("t5: from_pretrained must name the T5 checkpoint")
        if dtype not in _DTYPES:
            raise ValueError(f"t5: dtype {dtype} is not supported (torch.float32 or torch.bfloat16; computes in bfloat16)")
        self.from_pretrained = resolve_pretrained(from_pretrained, cache_dir)
        self.t5 = HFEmbedder(self.from_pretrained, max_length=model_max_length, shardformer=shardformer,
                             device_map=device, torch_dtype=torch.bfloat16)
        self._tokenizer = tokenizer
        self.y_embedder = None
        self.model_max_length = model_max_length
        self.output_dim = self.t5.config["d_model"]
        self.dtype = dtype

    @property
    def tokenizer(self):
        if self._tokenizer is None:
            from transformers import AutoTokenizer

            self._tokenizer = AutoTokenizer.from_pretrained(self.from_pretrained, local_files_only=True)
        return self._tokenizer

    @property
    def device(self) -> torch.device:
        return self.t5.shared.device

    def encode(self, text: list[str]) -> dict:
        enc = self.tokenizer(text, max_length=self.model_max_length, padding="max_length", truncation=True,
                             return_attention_mask=True, add_special_tokens=True, return_tensors="pt")
        ids = enc["input_ids"].to(self.device)
        mask = enc["attention_mask"].to(self.device, torch.int64)
        return dict(y=self.t5.encode(ids, mask)[:, None], mask=mask)

    def null(self, n: int) -> torch.Tensor:
        if self.y_embedder is None:
            raise RuntimeError("t5.null: the null caption is the denoiser's `y_embedder.y_embedding`; set "
                               "`text_encoder.y_embedder = model.y_embedder` first")
        return self.y_embedder.y_embedding[None].repeat(n, 1, 1)[:, None]
