"""One tiny denoise step of the osb200 STDiT3 on cuda:0, checked against the oracle (the only
place outside tests/ and bench.py's cpu_baseline that touches oracle/, as the checker)."""
import torch


def run_smoke():
    from tests.models import stdit3_inputs, stdit3_pair
    from tests.util import report

    assert torch.cuda.is_available(), "smoke() needs cuda:0"
    torch.cuda.set_device(0)
    prod, oracle, cfg = stdit3_pair("xs")
    inp = stdit3_inputs(cfg, 1, 8, 16, 16, device="cuda")
    with torch.no_grad():
        ref = oracle.cuda()(**inp)
        out = prod(**inp)
    torch.cuda.synchronize()
    r, _ = report("smoke STDiT3-XS/2 1x8x16x16", out, ref)
    assert out.shape == ref.shape and torch.isfinite(out).all()
    assert r < 2e-2, f"smoke parity failed: rel_l2={r}"
    import osb200

    print(f"smoke ok: osb200 launched {osb200.launch_count()} kernels")
