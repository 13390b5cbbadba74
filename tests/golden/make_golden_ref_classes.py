"""Fixture for the tests that compare with classes of the reference checkout (tests/golden/ref_classes.npz).

Run with the reference checkout available to oracle/ref_loader.py:  python tests/golden/make_golden_ref_classes.py

  * mmdit_{fused}_*: the reference's DoubleStreamBlock / SingleStreamBlock (mmdit/layers.py) executed by path in fp32 on
    the seeded parameters and inputs of tests/test_host_mmdit_cpu.py::test_processors_run_on_the_reference_own_blocks,
    plus the rel-L2 of the reference's own bf16 path (its noise floor).  The in-tree mirror draws identical parameters
    from the same seed (checked here), so the fixture stores outputs only: every TOKEN_STRIDE-th token, in float16.
  * posterior_*: the reference's DiagonalGaussianDistribution (hunyuan_vae/vae.py) on the inputs of
    tests/test_host_vae_cpu.py::test_posterior_distribution_matches_the_reference_class.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "open-sora_b200"))

from oracle import ref_loader  # noqa: E402
from tests.test_host_mmdit_cpu import TOKEN_STRIDE, mmdit_block_case  # noqa: E402
from tests.test_host_vae_cpu import posterior_inputs  # noqa: E402
from tests.util import rel_l2  # noqa: E402


def main():
    assert ref_loader.available(), "the reference checkout is needed to produce this fixture"
    out = {}
    R, _, _ = ref_loader.load_mmdit()
    from opensora.models.mmdit import layers as ours

    for fused in (True, False):
        dbl, sgl, pe, img, txt, vec = mmdit_block_case(R, fused)
        dbl_o, sgl_o, pe_o, img_o, txt_o, vec_o = mmdit_block_case(ours, fused)
        for a, b in ((dbl, dbl_o), (sgl, sgl_o)):
            pa, pb = dict(a.named_parameters()), dict(b.named_parameters())
            assert list(pa) == list(pb) and all(torch.equal(pa[k], pb[k]) for k in pa), "mirror parameters differ"
        assert torch.equal(pe, pe_o) and torch.equal(img, img_o) and torch.equal(txt, txt_o) and torch.equal(vec, vec_o)
        with torch.no_grad():
            ref_i, ref_t = dbl(img.float(), txt.float(), vec.float(), pe)
            ref_x = sgl(torch.cat((txt, img), 1).float(), vec.float(), pe)
            noise_i, _ = dbl.to(torch.bfloat16)(img, txt, vec, pe)
        tag = "fused" if fused else "split"
        out[f"mmdit_{tag}_img"] = ref_i[:, ::TOKEN_STRIDE].half().numpy()
        out[f"mmdit_{tag}_txt"] = ref_t[:, ::TOKEN_STRIDE].half().numpy()
        out[f"mmdit_{tag}_single"] = ref_x[:, ::TOKEN_STRIDE].half().numpy()
        out[f"mmdit_{tag}_bf16_floor"] = np.float64(rel_l2(noise_i.float(), ref_i))

    _, Rvae = ref_loader.load_hunyuan_vae()
    for i, (par, par2) in enumerate(posterior_inputs()):
        b, b2 = Rvae.DiagonalGaussianDistribution(par), Rvae.DiagonalGaussianDistribution(par2)
        sb = b.sample(torch.Generator().manual_seed(11))
        out[f"posterior{i}_mode"] = b.mode().numpy()
        out[f"posterior{i}_std"] = b.std.numpy()
        out[f"posterior{i}_logvar"] = b.logvar.numpy()
        out[f"posterior{i}_sample"] = sb.numpy()
        out[f"posterior{i}_kl"] = b.kl().numpy()
        out[f"posterior{i}_kl2"] = b.kl(b2).numpy()
        if par.ndim >= 4:
            out[f"posterior{i}_nll"] = b.nll(sb, list(range(1, par.ndim))).numpy()
    path = os.path.join(ROOT, "tests", "golden", "ref_classes.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
