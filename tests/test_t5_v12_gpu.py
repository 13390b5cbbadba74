"""The padding-masked T5 encoder and Open-Sora v1.2's "t5" text encoder on the H100: the tiny golden case and the full
24-layer T5-XXL shape with right-padded masks against the masked oracle (pinned on the CPU by transformers' golden) in
fp32 and in bf16 on the same device, the size of what the mask changes, and one prompt -> latent run of v1.2's
pipeline (T5 -> STDiT3-XS/2 -> RFLOW).  Each case prints its error, floor and ratio."""
import pytest
import torch

from tests.text_gpu_common import encoder_parity
from tests.util import rel_l2

pytestmark = pytest.mark.gpu


def _osb():
    import osb200

    osb200.init()
    return osb200


def test_masked_golden_case_on_device(tmp_path):
    _osb()
    from tests import text_fixtures as tf
    from tests.t5_masked_ref import t5_encode_masked
    from tests.t5_v12_common import golden
    from opensora.models.text.conditioner import HFEmbedder

    _, ids, mask, _ = golden()
    wb = {k: v.bfloat16().float() for k, v in tf.t5_weights(tf.T5_TINY, tf.SEED_T5).items()}
    emb = HFEmbedder(tf.write_checkpoint(str(tmp_path / "t5"), tf.T5_TINY, wb), max_length=300, device_map="cuda",
                     torch_dtype=torch.bfloat16)
    ids, mask = ids.cuda(), mask.cuda()
    torch.backends.cuda.matmul.allow_tf32 = False
    encoder_parity("T5 tiny masked 3x300", emb.encode(ids, mask), t5_encode_masked(wb, tf.T5_TINY, ids, mask),
                    t5_encode_masked(wb, tf.T5_TINY, ids, mask, torch.bfloat16), 5e-2)


def test_full_t5_xxl_masked_vs_oracle(tmp_path):
    _osb()
    from tests import text_fixtures as tf, text_gpu_common as G
    from tests.t5_masked_ref import t5_encode_masked
    from opensora.models.text.conditioner import _t5_shapes

    cfg = tf.T5_XXL
    w = G.device_weights(_t5_shapes(cfg), False, 5, cfg["d_model"])
    emb = G.build(str(tmp_path), cfg, w, False, 300)
    lens = [1, 17, 120, 300]
    gen = torch.Generator(device="cuda").manual_seed(11)
    ids = torch.randint(2, cfg["vocab_size"], (4, 300), generator=gen, device="cuda")
    mask = (torch.arange(300, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]).long()
    ids[torch.arange(4, device="cuda"), torch.tensor(lens, device="cuda") - 1] = 1   # eos
    ids[mask == 0] = 0                                  # pad
    out = emb.encode(ids, mask)
    unmasked = emb.encode(ids)
    torch.backends.cuda.matmul.allow_tf32 = False
    fp32 = t5_encode_masked(w, cfg, ids, mask)
    bf16 = t5_encode_masked(w, cfg, ids, mask, torch.bfloat16)
    # random 24-layer T5 weights grow the residual stream: the bf16 floor itself is about 0.11 here
    encoder_parity("T5-XXL masked 4x300", out, fp32, bf16, 0.15)
    bar = 1.1 * rel_l2(bf16.float(), fp32)
    for b, n in enumerate(lens[:2]):   # the short prompts' real tokens: without the mask they attend ~300 pads
        drop = rel_l2(unmasked[b, :n].float(), out[b, :n].float())
        print(f"T5-XXL prompt of {n} tokens: unmasked vs masked rel-L2 {drop:.3e}, bar {bar:.3e}")
        assert drop > 3 * bar, (n, drop, bar)


def test_prompt_to_latent_on_device(tmp_path):
    _osb()
    from tests.t5_v12_common import run_pipeline

    torch.backends.cuda.matmul.allow_tf32 = False
    out, ref, noise, seen, mask = run_pipeline(tmp_path, "cuda")
    assert len(seen) == 3 and all(torch.equal(m, torch.cat((mask, mask))) for m in seen)
    assert out.dtype == torch.bfloat16 and torch.isfinite(out.float()).all()
    r, rn = rel_l2(out.float(), ref), rel_l2(noise, ref)
    print(f"prompt -> latent on the device: rel-L2 {r:.3e}, bf16 floor {rn:.3e}")
    assert r < max(1.5 * rn, 1e-2) and r < 6e-2, (r, rn)
