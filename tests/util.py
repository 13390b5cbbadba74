"""Parity metrics shared by the tests (max-abs, rel-L2 against an fp32 reference), the golden fixtures and the
head-tile decoder and the self- and cross-attention cases of the head-tile tests."""
import math

import torch


def rel_l2(a: torch.Tensor, ref: torch.Tensor) -> float:
    a = a.double().flatten()
    ref = ref.double().flatten()
    return float((a - ref).norm() / ref.norm().clamp_min(1e-30))


def max_abs(a: torch.Tensor, ref: torch.Tensor) -> float:
    return float((a.double() - ref.double()).abs().max())


def report(name: str, a: torch.Tensor, ref: torch.Tensor) -> tuple[float, float]:
    r, m = rel_l2(a, ref), max_abs(a, ref)
    print(f"[parity] {name}: rel_l2={r:.3e} max_abs={m:.3e} ref_absmax={float(ref.abs().max()):.3e}")
    return r, m


# one bf16 rounding of an exact result has RMS relative error 2^-9/sqrt(3) ~ 1.1e-3
BF16_ONE_ROUNDING_REL_L2 = 2.0e-3


# ---- golden fixtures (tests/golden/*.npz) -----------------------------------------------------------------------------
# Random weights are not stored: a generator sets every parameter from a seed derived from its name (seeded_init) and
# the fixture keeps the name -> (seed key, parameter name, shape) manifest; load_golden regenerates the same values.
import json as _json  # noqa: E402
import os as _os  # noqa: E402
import zlib as _zlib  # noqa: E402

import numpy as _np  # noqa: E402

GOLDEN = _os.path.join(_os.path.dirname(_os.path.abspath(__file__)), "golden")
_SEEDED: dict = {}


def seeded_param(key: str, name: str, shape) -> torch.Tensor:
    """Deterministic fp32 value of parameter `name` under seed key `key`: norm weights / scales 1 + 0.2 N(0,1), other
    vectors 0.1 N(0,1), matrices and kernels U(-1, 1) / sqrt(fan_in) (the spread of torch's default Linear / Conv init)."""
    shape = tuple(int(s) for s in shape)
    g = torch.Generator().manual_seed(_zlib.crc32(key.encode()))
    leaf = name.rsplit(".", 1)[-1]
    if len(shape) == 1:
        x = torch.randn(shape, generator=g)
        return 1.0 + 0.2 * x if (leaf == "scale" or (leaf == "weight" and "norm" in name)) else 0.1 * x
    x = torch.rand(shape, generator=g) * 2.0 - 1.0
    return x * (x.numel() // shape[0]) ** -0.5


def seeded_init(module, prefix: str) -> None:
    """Golden generators: overwrite every parameter of `module` with seeded_param(prefix.name)."""
    with torch.no_grad():
        for n, p in module.named_parameters():
            p.copy_(seeded_param(f"{prefix}.{n}", n, p.shape))
            _SEEDED[p.data_ptr()] = (f"{prefix}.{n}", n)


def save_golden(path: str, out: dict, half=()) -> None:
    """Write `out` to `path`: seeded parameters as manifest entries, keys in `half` as float16, the rest as float32."""
    arrays, params = {}, {}
    for k, t in out.items():
        t = t.detach()
        seeded = _SEEDED.get(t.data_ptr()) if t.numel() else None
        if seeded is not None:
            params[k] = [seeded[0], seeded[1], list(t.shape)]
        else:
            arrays[k] = t.float().numpy().astype(_np.float16 if k in half else _np.float32)
    arrays["__seeded_params__"] = _np.array(_json.dumps(params, sort_keys=True))
    _np.savez_compressed(path, **arrays)


def load_golden(name: str) -> dict:
    """tests/golden/<name> as {key: fp32 tensor}, seeded parameters regenerated."""
    z = _np.load(_os.path.join(GOLDEN, name))
    G = {k: torch.from_numpy(z[k].astype(_np.float32)) for k in z.files if k != "__seeded_params__"}
    if "__seeded_params__" in z.files:
        for k, (key, n, shape) in _json.loads(str(z["__seeded_params__"])).items():
            G[k] = seeded_param(key, n, shape)
    return G


# ---- head tiles (tiles.cuh) ------------------------------------------------------------------------------------------
def _cuda():
    """cuda:0, or a skip of the calling test when there is no CUDA device."""
    if not torch.cuda.is_available():
        import pytest

        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _rms(x, w, eps=1e-6):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def _rope(x, cos, sin):
    """interleaved pairs (2i, 2i+1); x [..., L, D], cos/sin [L, D/2]"""
    a, b = x[..., 0::2], x[..., 1::2]
    out = torch.empty_like(x)
    out[..., 0::2] = a * cos - b * sin
    out[..., 1::2] = b * cos + a * sin
    return out


def read_tiles(tiles, kind):
    """Decode one kind of a HeadTiles buffer back to a dense [rows, heads*D] bf16 tensor (inverse of tiles.cuh)."""
    m, D, H = tiles.map, tiles.head_dim, tiles.heads
    DP = -(-D // 16) * 16
    TR = m.tile_rows
    dev = tiles.buf.device
    rows = torch.arange(tiles.rows, device=dev)
    if m.mode == 0:
        seq, pos = rows // m.L, rows % m.L
    else:
        b, rem = rows // (m.T * m.S), rows % (m.T * m.S)
        pos, seq = rem // m.S, b * m.S + rem % m.S
    if m.G > 1:
        tile, r = seq // m.G, (seq % m.G) * m.L + pos
    else:
        tile, r = seq * m.tps + pos // TR, pos % TR
    raw = tiles.buf[kind * tiles.kind_stride:(kind + 1) * tiles.kind_stride].view(torch.int16)
    out = torch.empty(tiles.rows, H * D, dtype=torch.int16, device=dev)
    main = D // 64
    for h in range(H):
        base = (h * tiles.head_stride + tile * tiles.tile_bytes) // 2          # in int16 elements
        for u in range(D // 8):
            if u < main * 8:
                off = (u // 8) * TR * 64 + (r // 8) * 512 + (r % 8) * 64 + (((u % 8) ^ (r % 8)) * 8)
            else:
                off = main * TR * 64 + (r // 8) * 128 + (u - main * 8) * 64 + (r % 8) * 8
            idx = (base + off)[:, None] + torch.arange(8, device=dev)[None]
            out[:, h * D + u * 8:h * D + u * 8 + 8] = raw[idx]
    return out.view(torch.bfloat16)


def self_case(mode, B, T, S, H, D, seed=0, general=False, transposed=False):
    """One STDiT3-style self-attention: tokens frame-major [B, T, S]; mode 0 attends over S, mode 1 over T (with RoPE)."""
    import osb200 as osb

    dev = _cuda()
    g = torch.Generator(device="cpu").manual_seed(seed)
    C = H * D
    R = B * T * S
    x = (torch.randn(R, C, generator=g) * 1.0).to(torch.bfloat16).to(dev)
    w = (torch.randn(3 * C, C, generator=g) / math.sqrt(C)).to(torch.bfloat16).to(dev)
    bias = (torch.randn(3 * C, generator=g) * 0.1).to(torch.bfloat16).to(dev)
    qn = (1.0 + 0.2 * torch.randn(D, generator=g)).to(torch.bfloat16).to(dev)
    kn = (1.0 + 0.2 * torch.randn(D, generator=g)).to(torch.bfloat16).to(dev)
    L = S if mode == 0 else T
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2).float() / D))
    ang = torch.arange(L).float()[:, None] * inv[None]
    cos, sin = ang.cos().contiguous().to(dev), ang.sin().contiguous().to(dev)
    tm = osb.tile_map(0, S) if mode == 0 else osb.tile_map(1, T, S, T)
    x_in, out_map = x, None
    if transposed:   # temporal sequences as contiguous row blocks ([B, S, T] stream), output still frame-major
        assert mode == 1
        x_in = x.view(B, T, S, C).transpose(1, 2).reshape(R, C).contiguous()
        tm, out_map = osb.tile_map(0, T), tm
    tiles = osb.HeadTiles(R, tm, 3, H, D, dev)
    osb.gemm_head_tiles(x_in, w, bias, tiles, nkinds=3, norm_w=(qn, kn, None), rope=(cos, sin) if mode == 1 else None,
                        rope_kinds=0b011, general=general)
    out = torch.full((R, C), float("nan"), dtype=torch.bfloat16, device=dev)
    nseq = B * T if mode == 0 else B * S
    osb.attn_tiles(tiles, tiles, out, Lk=L, num_seqs=nseq, out_map=out_map)
    torch.cuda.synchronize()

    # fp32 restatement
    qkv = (x.float() @ w.float().t() + bias.float()).view(B, T, S, 3, H, D)
    q, k, v = qkv[..., 0, :, :], qkv[..., 1, :, :], qkv[..., 2, :, :]
    q, k = _rms(q, qn.float()), _rms(k, kn.float())
    if mode == 0:
        q, k, v = (t.permute(0, 1, 3, 2, 4) for t in (q, k, v))          # [B, T, H, S, D]
    else:
        q, k, v = (t.permute(0, 2, 3, 1, 4) for t in (q, k, v))          # [B, S, H, T, D]
        q, k = _rope(q, cos, sin), _rope(k, cos, sin)
    # what the tiles must hold (token layout)
    def back(t):
        t = t.permute(0, 1, 3, 2, 4) if mode == 0 else t.permute(0, 3, 1, 2, 4)
        return t.reshape(R, C)
    for kind, ref in enumerate((q, k, v)):
        got = read_tiles(tiles, kind).float()
        if transposed:
            got = got.view(B, S, T, C).transpose(1, 2).reshape(R, C)
        e = rel_l2(got, back(ref))
        assert e < 2.5e-3, (kind, e)
    # attention on the bf16-rounded operands the kernel sees
    qb, kb, vb = (t.to(torch.bfloat16).float() for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qb, kb, vb)
    ref = back(o)
    assert torch.isfinite(out.float()).all()
    e = rel_l2(out.float(), ref)
    assert e < 5e-3, e
    return e


def cross_case(B, N, Ly, lens, H):
    """STDiT3-style cross-attention: B samples of N query tokens against Ly text tokens of which the first lens[b]
    are valid, the keys and values of several blocks in one head-tile set (checked for the first and the last block)."""
    import osb200 as osb

    dev = _cuda()
    D = 72
    C = H * D
    g = torch.Generator().manual_seed(11)
    xq = torch.randn(B * N, C, generator=g).to(torch.bfloat16).to(dev)
    y = torch.randn(B * Ly, C, generator=g).to(torch.bfloat16).to(dev)
    wq = (torch.randn(C, C, generator=g) / math.sqrt(C)).to(torch.bfloat16).to(dev)
    bq = (torch.randn(C, generator=g) * 0.1).to(torch.bfloat16).to(dev)
    nblk = 3                                                      # kv_linear of several blocks in one GEMM
    wkv = (torch.randn(nblk * 2 * C, C, generator=g) / math.sqrt(C)).to(torch.bfloat16).to(dev)
    bkv = (torch.randn(nblk * 2 * C, generator=g) * 0.1).to(torch.bfloat16).to(dev)
    kv_lens = torch.tensor(lens, dtype=torch.int32, device=dev)
    qt = osb.HeadTiles(B * N, osb.tile_map(0, N), 1, H, D, dev)
    kt = osb.HeadTiles(B * Ly, osb.tile_map(0, Ly, keys_only=True), 2 * nblk, H, D, dev)
    osb.gemm_head_tiles(xq, wq, bq, qt, nkinds=1)
    osb.gemm_head_tiles(y, wkv, bkv, kt, nkinds=2)
    q = (xq.float() @ wq.float().t() + bq.float()).to(torch.bfloat16).float().view(B, N, H, D).permute(0, 2, 1, 3)
    kvf = (y.float() @ wkv.float().t() + bkv.float()).to(torch.bfloat16).float().view(B, Ly, nblk, 2, H, D)
    for blk in (0, 2):
        out = torch.full((B * N, C), float("nan"), dtype=torch.bfloat16, device=dev)
        osb.attn_tiles(qt, kt, out, q_kind=0, k_kind=2 * blk, v_kind=2 * blk + 1, Lk=Ly, num_seqs=B, kv_lens=kv_lens)
        assert torch.isfinite(out.float()).all()
        for b in range(B):
            n = lens[b]
            got = out[b * N:(b + 1) * N].float()
            if n == 0:
                assert (got == 0).all()
                continue
            k = kvf[b, :n, blk, 0].permute(1, 0, 2)
            v = kvf[b, :n, blk, 1].permute(1, 0, 2)
            ref = torch.nn.functional.scaled_dot_product_attention(q[b], k, v).permute(1, 0, 2).reshape(N, C)
            e = rel_l2(got, ref)
            assert e < 5e-3, (blk, b, e)
