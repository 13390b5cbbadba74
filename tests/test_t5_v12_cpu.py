"""Open-Sora v1.2's T5 text encoder (`type="t5"`, opensora/models/text_encoder/t5.py) and the padding mask of the T5
encoder without a GPU: the masked T5 reference (tests/t5_masked_ref.py) and the host model on the binding stand-in against the golden of transformers'
T5EncoderModel(input_ids, attention_mask) (tests/golden/make_golden_t5_masked.py), mask refusals, the registry path of
a v1.2 config, checkpoint resolution, and one prompt -> latent run of the v1.2 pipeline (T5 -> STDiT3-XS/2 -> RFLOW)."""
import json
import os

import numpy as np
import pytest
import torch

from tests import text_fixtures as tf
from tests.t5_v12_common import MaskingToyTokenizer, golden as _golden, t5_dir as _t5_dir, t5_oracle
from tests.util import rel_l2


def _floor(ids, mask):
    return t5_oracle(ids, mask, torch.bfloat16)


def _bar(floor_out, golden):
    # the bar of the existing text tests: the bf16 oracle's error, + 25% + 2e-3 for the fused epilogues' rounding points
    return 1.25 * rel_l2(floor_out.float(), golden) + 2e-3


# ---- oracle and host model against transformers ------------------------------------------------------------------
def test_masked_reference_matches_transformers_golden():
    from oracle import text_oracle as O
    from tests.t5_masked_ref import t5_encode_masked

    _, ids, mask, out = _golden()
    assert mask.sum(1).tolist() == [1, 7, 300]
    w = tf.t5_weights(tf.T5_TINY, tf.SEED_T5)
    np.testing.assert_allclose(t5_encode_masked(w, tf.T5_TINY, ids, mask).numpy(), out.numpy(), rtol=2e-5, atol=2e-5)
    # with nothing masked it is the pinned text oracle, bit for bit, in fp32 and in bf16
    ones = torch.ones_like(mask)
    for dt in (torch.float32, torch.bfloat16):
        assert torch.equal(t5_encode_masked(w, tf.T5_TINY, ids, ones, dt), O.t5_encode(w, tf.T5_TINY, ids, dt))


def test_masked_host_model_on_stand_in_vs_golden(fake_osb, tmp_path):
    from opensora.models.text.conditioner import HFEmbedder

    _, ids, mask, golden = _golden()
    emb = HFEmbedder(_t5_dir(tmp_path), max_length=300, torch_dtype=torch.bfloat16)
    out = emb.encode(ids, mask)
    assert out.shape == (3, 300, 128) and out.dtype == torch.bfloat16
    floor = _floor(ids, mask)
    unmasked = emb.encode(ids)
    for b in range(3):
        err, bar = rel_l2(out[b].float(), golden[b]), _bar(floor[b], golden[b])
        assert err <= bar, (b, err, bar)
        if b < 2:   # pad-heavy prompts: without the mask the ~300 pad keys swamp every layer's attention
            drop = rel_l2(unmasked[b].float(), golden[b])
            assert drop > 10 * bar, (b, drop, bar)
        else:       # no pads: the mask changes nothing
            assert torch.equal(unmasked[b], out[b])
    # the mask rides on the attention launch: no extra launches per layer
    names = [c[0] for c in fake_osb.calls]
    assert names.count("attn_short") == 2 * 2 and names.count("gemm") == 2 * 4 * 2


@pytest.mark.parametrize("case", ["left_padded", "hole", "empty_row", "value_2", "shape"])
def test_mask_refusals(fake_osb, tmp_path, case):
    from opensora.models.text.conditioner import HFEmbedder

    emb = HFEmbedder(_t5_dir(tmp_path), max_length=16)
    ids = torch.full((2, 16), 5, dtype=torch.long)
    m = torch.ones(2, 16, dtype=torch.long)
    m[1, 9:] = 0
    match = "right-padded"
    if case == "left_padded":
        m[0, :4] = 0
    elif case == "hole":
        m[0, 3] = 0
    elif case == "empty_row":
        m[1] = 0
        match = r"rows \[1\] have no real token"
    elif case == "value_2":
        m[0, 0] = 2
    else:
        m, match = m[:, :15], "shape"
    n0 = fake_osb.launch_count()
    with pytest.raises(ValueError, match=match):
        emb.encode(ids, m)
    assert fake_osb.launch_count() == n0


def test_clip_refuses_a_mask(fake_osb, tmp_path):
    from opensora.models.text.conditioner import HFEmbedder

    d = tf.write_checkpoint(str(tmp_path / "openai/clip"), tf.CLIP_TINY, tf.clip_weights(tf.CLIP_TINY, tf.SEED_CLIP))
    emb = HFEmbedder(d, max_length=77)
    ids = torch.full((1, 77), 5, dtype=torch.long)
    with pytest.raises(ValueError, match="T5 only"):
        emb.encode(ids, torch.ones(1, 77, dtype=torch.long))


# ---- the v1.2 encoder ------------------------------------------------------------------------------------------------
def _v12_cfg(tmp_path):
    return dict(type="t5", from_pretrained=_t5_dir(tmp_path), model_max_length=300, shardformer=True)


def test_v12_config_builds_and_encodes(fake_osb, tmp_path):
    from opensora.models.text_encoder import T5Encoder
    from opensora.registry import MODELS, build_module

    text, ids, mask, golden = _golden()
    t5 = build_module(_v12_cfg(tmp_path), MODELS, device="cpu", tokenizer=MaskingToyTokenizer())
    assert isinstance(t5, T5Encoder)
    assert t5.model_max_length == 300 and t5.output_dim == 128 and t5.dtype == torch.float32 and t5.y_embedder is None
    res = t5.encode(text)
    assert set(res) == {"y", "mask"}
    assert res["y"].shape == (3, 1, 300, 128) and res["y"].dtype == torch.bfloat16
    assert res["mask"].dtype == torch.int64 and torch.equal(res["mask"], mask)
    assert torch.equal(res["y"][:, 0], t5.t5.encode(ids, mask))
    err = rel_l2(res["y"][:, 0].float(), golden)
    assert err <= _bar(_floor(ids, mask), golden), err
    # null(): the denoiser's caption embedding, once the v1.2 script has handed it over
    with pytest.raises(RuntimeError, match="y_embedder"):
        t5.null(2)
    cap = torch.nn.Module()
    cap.register_buffer("y_embedding", torch.randn(300, 128).bfloat16())
    t5.y_embedder = cap
    y_null = t5.null(2)
    assert y_null.shape == (2, 1, 300, 128) and torch.equal(y_null[1, 0], cap.y_embedding)
    # bf16 is accepted too and computes the same; other dtypes are refused
    t5b = build_module(_v12_cfg(tmp_path), MODELS, device="cpu", dtype=torch.bfloat16, tokenizer=MaskingToyTokenizer())
    assert t5b.dtype == torch.bfloat16 and torch.equal(t5b.encode(text)["y"], res["y"])
    with pytest.raises(ValueError, match="float16"):
        build_module(_v12_cfg(tmp_path), MODELS, device="cpu", dtype=torch.float16)


def _write_bin_index(path, weights):
    """DeepFloyd/t5-v1_1-xxl's layout: encoder-only weights (embed_tokens stored beside shared) in two .bin shards
    named by pytorch_model.bin.index.json."""
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as fh:
        json.dump(dict(tf.T5_TINY, architectures=["T5EncoderModel"]), fh)
    w = dict(weights, **{"encoder.embed_tokens.weight": weights["shared.weight"]})
    keys = sorted(w)
    wm = {}
    for i, part in enumerate((keys[: len(keys) // 2], keys[len(keys) // 2:])):
        name = f"pytorch_model-{i + 1:05d}-of-00002.bin"
        torch.save({k: w[k] for k in part}, os.path.join(path, name))
        wm.update({k: name for k in part})
    with open(os.path.join(path, "pytorch_model.bin.index.json"), "w") as fh:
        json.dump({"metadata": {}, "weight_map": wm}, fh)


def test_hub_cache_and_bin_index_checkpoint(fake_osb, tmp_path, monkeypatch):
    """`from_pretrained="DeepFloyd/t5-v1_1-xxl"` resolves to the cached snapshot under `cache_dir` (no download), and
    its .bin index layout loads."""
    from opensora.registry import MODELS, build_module

    text, ids, mask, golden = _golden()
    cache = tmp_path / "hf"
    _write_bin_index(str(cache / "models--DeepFloyd--t5-v1_1-xxl" / "snapshots" / "0123abc"),
                     tf.t5_weights(tf.T5_TINY, tf.SEED_T5))
    for var in ("HF_HOME", "HF_HUB_CACHE"):
        monkeypatch.setenv(var, str(tmp_path / "empty"))
    t5 = build_module(dict(type="t5", from_pretrained="DeepFloyd/t5-v1_1-xxl", model_max_length=300, shardformer=True,
                           cache_dir=str(cache)), MODELS, device="cpu", tokenizer=MaskingToyTokenizer())
    err = rel_l2(t5.encode(text)["y"][:, 0].float(), golden)
    assert err <= _bar(_floor(ids, mask), golden), err
    with pytest.raises(FileNotFoundError, match="DeepFloyd/t5-v1_1-xl"):
        build_module(dict(type="t5", from_pretrained="DeepFloyd/t5-v1_1-xl", cache_dir=str(cache)), MODELS, device="cpu")


def test_prompt_to_latent_v12_pipeline(fake_osb, tmp_path):
    """v1.2's inference wiring on the stand-in (tests/t5_v12_common.py), at the bar of test_rflow_sampler_drives_the_model."""
    from tests.t5_v12_common import run_pipeline

    out, ref, noise, seen, mask = run_pipeline(tmp_path, "cpu")
    # both CFG branches see the prompt's caption mask (the null caption is cut to the prompt's length)
    assert len(seen) == 3 and all(torch.equal(m, torch.cat((mask, mask))) for m in seen)
    assert out.dtype == torch.bfloat16
    r, rn = rel_l2(out.float(), ref), rel_l2(noise, ref)
    print(f"prompt -> latent: rel-L2 {r:.3e}, bf16 floor {rn:.3e}")
    assert r < max(1.5 * rn, 1e-2) and r < 6e-2, (r, rn)
    assert [c[0] for c in fake_osb.calls].count("cfg_euler") == 3
