"""Attention cases whose output is known exactly, for bit-identical tests of `attn_tiles`, `attn_tiles_fp8`, `attn_short`,
`attn_fp8`, `attn_fp8_blocks`, `attn_short_bias` and `attn_frames`.

A rel-L2 bound cannot see a masking or indexing error: one key too many or too few among hundreds moves an output row by
about |v| / L, far inside any whole-tensor bar.  These cases remove the rounding instead of bounding it
(tests/exact_gemm.py does the same for the GEMMs): every query row gets one winning key among the keys it may see, and
the winner's score beats every other visible key by at least MARGIN = 160 log2 units while staying within 2^10 of 0.
Then every losing exp2 is exactly 0 in fp32, the winner's p is 1 up to the rounding residue of its own score (< 2^-13),
bf16(p) = 1, and the output row is the winner's value row.  Every value is +-{1, 1.25, 1.5, 1.75} x 2^e (at most three
significant bits), at least 2^-9 relative away from a bf16 rounding boundary, so the kernels' few fp32 ulps (1 / l,
ex2.approx of a residue) round back to it: the output must equal the winning value row bit for bit.  A tie mode gives a
row k = 2 or 4 winners with identical keys in different key blocks; its output is the mean of their value rows, which
`check_budget` proves exact in bf16 (the running maximum stops changing: alpha = 1).

Scores.  Key j carries an address code c_j: one +-1 in each of three channel groups of gs = (D - 1) // 3 channels, the
symbols of the three groups being (a, b, (a + b) mod 2 gs), so two different codes agree in at most one group and
c_i . c_j <= 1 for i != j while c . c = 3.  A query row is alpha c_w for its winner w: the winner scores 3 alpha, every
other code at most alpha.  Channel 3 gs is +1 in every real key; a "negative" query row puts -8 alpha there, so every
visible score is negative (the winner -5 alpha) and a zero-filled pad key slot, scoring 0, would win if it leaked.
alpha x softmax_scale x log2(e) lies in [163, 185] for D in {64, 72, 128, 512}, so the margin is >= 160 and
|winner| <= 5 x 185 < 2^10.  Every nonzero of a q row is +-alpha or -8 alpha and of a k row +-1, +-2 or 1: the e4m3 per-row
codes of the FP8 paths are exact (448, 224, 56).

Decoys.  Keys a row must not see get twice the code of a winner of that row's group (they would beat it by 3 alpha if
they leaked) and sit where an off-by-one mask would leak them: the slots just past kv_lens, the first keys of the
neighbouring packed sequence, the first keys of the next frame.  Causal rows get theirs at j = i + 1.  A leak replaces a
whole output row instead of nudging it.

QK-norm and RoPE.  `short_case(..., norm_split=, rope=)` designs q / k in post-RoPE space and undoes RoPE with
quarter-turn tables (cos, sin in {0, +-1}, a different turn per position and pair), so RoPE is an exact signed
permutation in either pairing and a row rotated for the wrong position loses its winner.  RMSNorm uses constant weights
per stream: w for tokens below norm_split, 2 w above, for q and for k.  Every key row has the same norm, so all staged
keys of a stream are +-rho_k, and every q row is +-rho_q: the scores keep the code arithmetic, scaled by stream.
Winners are keys of the second stream, and every winning code has a copy in the first stream that scores half as much:
a key staged with the other stream's weight turns that pair into an exact tie, which moves the output row.  Rows are
all "positive" here (pad keys are covered by the cases without norm).  check_budget emulates the staging in fp64 and
allows the kernel's rsqrt one bf16 ulp on every staged value.

Values.  Per (sequence, head, channel) an exponent E_max in [-3, 1], reached in one 128-key block; the other blocks get
E in [E_max - 2, E_max].  Entries are +-m 2^e with e in [E - 3, E], and one entry +-1.75 x 2^E is planted in every
(128-key block, channel), never on a tied winner.  Every FP8 value scale group (per channel over the sequence for
`attn_fp8`, over a key tile for `attn_tiles_fp8`: key tiles are 128-key blocks or whole short sequences) therefore has
amax 1.75 x 2^E, s_v = 2^(E - 8) exactly, and every code is exact.  E varies by head, channel and key block, so a value
read with the wrong scale is off by a power of two.

`check_budget` proves all of this in fp64 before anything runs, from the operands themselves and a restatement of the
visibility rules of include/osb200.h that shares nothing with the kernels: kv_lens, separate (packed) sequences, the
relative-position bias (-inf masks), the frame-causal predicate with q_frame0, and pad key slots.  It raises
BudgetError on any violation.  Builders run on `device` from a seeded generator on that device."""
import copy
import math

import torch

from tests.exact_gemm import BudgetError, assert_bits, first_mismatch  # noqa: F401  (re-exported for the tests)

E4M3 = torch.float8_e4m3fn
LOG2E = 1.4426950408889634
MARGIN = 160.0              # log2 units between the winner and any other visible key
WIN_MAX = 1024.0            # |winner score| in log2 units: keeps the rounding residue of s * scale below 2^-13
ALPHA = {64: 1024.0, 72: 1024.0, 128: 1280.0, 512: 2560.0}
NEG = -8.0                  # the negative rows' entry in the all-ones key channel (in units of alpha)
FILLERS = 64                # codes reserved for keys that never win
REF_TOL = 2.0 ** -30        # fp64 dense softmax vs the expected rows
PAD = 8                     # sentinel columns on each side of sliced outputs
SENTINEL = -7.0


# ---- codes ------------------------------------------------------------------------------------------------------------
def n_codes(D):
    return (2 * ((D - 1) // 3)) ** 2


def code_vectors(ids, D):
    """Unit code vectors [..., D] of code ids [...] (channel 3 gs, the all-ones key channel, left 0)."""
    gs = (D - 1) // 3
    n = 2 * gs
    a, b = ids // n, ids % n
    syms = torch.stack((a, b, (a + b) % n), -1)
    pos = syms % gs + gs * torch.arange(3, device=ids.device)
    sign = (1 - 2 * (syms // gs)).float()
    out = torch.zeros(*ids.shape, D, device=ids.device)
    out.scatter_(-1, pos, sign)
    return out


def _randint(g, hi, shape):
    """Uniform integers in [0, hi) (hi a tensor broadcastable to shape, or an int), from g on its device."""
    r = torch.randint(0, 1 << 30, shape, generator=g, device=g.device)
    return r % hi


# ---- visibility (include/osb200.h, restated) ---------------------------------------------------------------------------
def bias_rel(case, r0, r1):
    """[Hb, r1 - r0, Lk] fp32: bias[h, j - i + Lq - 1] of rows i in [r0, r1)."""
    j = torch.arange(case.Lk, device=case.bias.device)
    i = torch.arange(r0, r1, device=case.bias.device)
    return case.bias.view(-1, case.Lq + case.Lk - 1)[:, j[None] - i[:, None] + case.Lq - 1]


def visible_pairs(case, s, i, j):
    """bool [..., Hb] for broadcastable sequence s, query row i and key j of that sequence."""
    ok = j < case.Lk
    if case.kv_lens is not None:
        ok = ok & (j < case.kv_lens.to(j.device).long()[s])
    if case.frames is not None:
        hw, f0 = case.frames
        ok = ok & (j < torch.clamp((f0 + i // hw + 1) * hw, max=case.Lk))
    ok = ok[..., None]
    if case.bias is not None:
        b = case.bias.view(-1, case.Lq + case.Lk - 1)[:, (j - i + case.Lq - 1).clamp(0, case.Lq + case.Lk - 2)]
        ok = ok & torch.isfinite(b).movedim(0, -1)
    return ok


def visible(case, s0, s1, r0, r1):
    """[s1 - s0, Hb, r1 - r0, Lk] bool: may query row i of sequence s see key j of the same sequence.  Keys of other
    sequences are never visible, whatever tile they share."""
    dev = case.q.device
    s = torch.arange(s0, s1, device=dev)[:, None, None]
    i = torch.arange(r0, r1, device=dev)[None, :, None]
    j = torch.arange(case.Lk, device=dev)[None, None, :]
    return visible_pairs(case, s, i, j).movedim(-1, 1)


def _units(case):
    """q / alpha and k as fp64, checked to be small integers: their dot products are exact in any format."""
    qu = case.q.double() / case.alpha
    ku = case.k.double()
    for name, u in (("q / alpha", qu), ("k", ku)):
        if not bool((u == u.round()).all()) or float(u.abs().max()) > 8:
            raise BudgetError(f"{name} must hold integers of magnitude <= 8")
    return qu, ku


def _dot(a, b):
    """a @ b^T of small-integer operands, exact: on CUDA bf16 tensor cores whose bf16 output holds every integer up to
    2^8, used only when sum |a| x max |b| proves |dot| <= 2^8 (the designs reach 14); fp64 otherwise."""
    if a.is_cuda and float(a.abs().sum(-1).max()) * float(b.abs().max()) <= 256:
        return (a.to(torch.bfloat16) @ b.to(torch.bfloat16).transpose(-1, -2)).double()
    return a.double() @ b.double().transpose(-1, -2)


def rope_rows(x, cos, sin, half, inverse=False):
    """RoPE (or its inverse) of fp64 rows x [..., L, D] with tables [L, D/2] whose entries are 0 or +-1 (a quarter turn
    per position and pair): a signed permutation, exact in any format.  half: pairs (i, i + D/2), else (2i, 2i + 1)."""
    c, s_ = cos.double(), (-sin if inverse else sin).double()
    D = x.shape[-1]
    a, b = (x[..., :D // 2], x[..., D // 2:]) if half else (x[..., 0::2], x[..., 1::2])
    a2, b2 = a * c - b * s_, b * c + a * s_
    return torch.cat((a2, b2), -1) if half else torch.stack((a2, b2), -1).flatten(-2)


def staged(case):
    """The bf16 q / k rows the kernels stage (fp64 [nseq, H, L, D]): RMSNorm with the weight of the token's stream
    (positions >= norm_split use the second pair), RoPE by position, one rounding."""
    st = case.stage
    out = []
    for x, w, w2 in ((case.q, st["qw"], st["qw2"]), (case.k, st["kw"], st["kw2"])):
        x = x.double()
        L = x.shape[2]
        r = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + st["eps"])
        wt = torch.where((torch.arange(L, device=x.device) >= st["split"])[:, None], w2.double()[None], w.double()[None])
        x = x * r * wt
        if st["cos"] is not None:
            x = rope_rows(x, st["cos"][:L], st["sin"][:L], st["half"])
        out.append(x.to(torch.bfloat16).double())
    return out


def _chunks(case):
    rows = max(1, min(case.Lq, (1 << 24) // max(1, case.H * case.Lk)))
    for s in range(case.nseq):
        for r0 in range(0, case.Lq, rows):
            yield s, r0, min(case.Lq, r0 + rows)


def _operands(case):
    """(q, k, factor): score = q . k x factor in log2 units.  Without QK-norm / RoPE q / alpha and k themselves (small
    integers, exact dots); with them the staged rows."""
    if case.stage is not None:
        qs, ks = staged(case)
        return qs, ks, case.scale * LOG2E
    qu, ku = _units(case)
    return qu, ku, case.alpha * case.scale * LOG2E


def scores(case, s, r0, r1, qu, ku, factor):
    """fp64 [1, H, r, Lk] scores in log2 units of rows [r0, r1) of sequence s; -inf where not visible."""
    S = _dot(qu[s:s + 1, :, r0:r1], ku[s:s + 1]) * factor
    if case.bias is not None:
        S = S + bias_rel(case, r0, r1).double()[None] * LOG2E
    return S.masked_fill(~visible(case, s, s + 1, r0, r1), -math.inf)


def _three_bits(name, x):
    m, _ = torch.frexp(x.double().abs())
    if not bool(((x == 0) | (m == 0.5) | (m == 0.625) | (m == 0.75) | (m == 0.875)).all()):
        raise BudgetError(f"{name}: every value must be 0 or +-{{1, 1.25, 1.5, 1.75}} x 2^e")


def check_budget(case):
    """Proves in fp64, before anything runs, that the case's output is exact: every row with a visible key has 1, 2 or 4
    tied winners, a margin >= MARGIN to every other visible key and |winner| <= WIN_MAX (log2 units); the mean of the
    winners' value rows is exact in bf16; every decoy is invisible to its row and would beat or tie its winner.  Sets
    case.expected (fp64 [nseq, H, Lq, D]) and case.winners (max tie count).  Raises BudgetError on any violation."""
    qu, ku, factor = _operands(case)
    # staged rows: the kernel's rsqrt may move a staged value by one bf16 ulp (2^-8 relative) from this emulation
    slack = 2.0 ** -7 if case.stage is not None else 0.0
    _three_bits("v", case.v)
    v = case.v.double()
    exp = torch.zeros(case.nseq, case.H, case.Lq, case.D, dtype=torch.float64, device=case.q.device)
    M = torch.full((case.nseq, case.H, case.Lq), -math.inf, dtype=torch.float64, device=case.q.device)
    ties = 0
    for s, r0, r1 in _chunks(case):
        S = scores(case, s, r0, r1, qu, ku, factor)[0]                       # [H, r, Lk]
        top = S.topk(min(5, case.Lk), dim=-1)
        m = top.values[..., 0]
        live = m > -math.inf
        win = (top.values == m[..., None]) & live[..., None]
        n = win.sum(-1)
        if bool((n[live] > 4).any()) or bool((n[live] == 3).any()):
            raise BudgetError(f"sequence {s}: a row has {int(n.max())} tied winners (1, 2 or 4 allowed)")
        second = torch.where(win, -math.inf, top.values).amax(-1)
        margin = m - second - slack * (m.abs() + torch.where(second > -math.inf, second.abs(), 0.0))
        if bool((live & (margin < MARGIN)).any()):
            raise BudgetError(f"sequence {s}: a winner beats another visible key by only {float(margin[live].min()):.3g} "
                              f"log2 units (< {MARGIN})")
        if bool((m[live].abs() > WIN_MAX).any()):
            raise BudgetError(f"sequence {s}: a winning score reaches {float(m[live].abs().max()):.4g} log2 units "
                              f"(> {WIN_MAX})")
        vw = v[s][torch.arange(case.H, device=v.device)[:, None, None], top.indices]   # [H, r, 5, D]
        mean = (vw * win[..., None]).sum(-2) / n.clamp(min=1)[..., None]
        if not bool((mean.to(torch.bfloat16).double() == mean).all()):
            raise BudgetError(f"sequence {s}: the mean of tied value rows is not exact in bf16")
        exp[s, :, r0:r1] = mean
        M[s, :, r0:r1] = m
        ties = max(ties, int(n.max()))
    if case.decoys is not None and len(case.decoys):
        sq, row, sk, key = case.decoys.unbind(1)
        d = (qu[sq, :, row] * ku[sk, :, key]).sum(-1) * factor                 # [nd, H]
        same = sq == sk
        if bool((visible_pairs(case, sq, row, key) & same[:, None]).any()):
            raise BudgetError("a decoy key is visible to the row it is planted for")
        if case.bias is not None:
            b = case.bias.view(-1, case.Lq + case.Lk - 1)[:, (key - row + case.Lq - 1).clamp(0, case.Lq + case.Lk - 2)]
            b = torch.where(torch.isfinite(b), b, 0.0)    # a -inf bias is the mask: a leak ignores it
            d = d + torch.where(same[:, None], b.t().double() * LOG2E, 0.0)
        if not bool((d >= M[sq, :, row]).all()):
            raise BudgetError("a decoy would neither beat nor tie its row's winner")
    case.expected, case.winners = exp, ties


def reference(case, leak=None):
    """fp64 dense masked softmax(q k^T scale + bias) v, [nseq, H, Lq, D], computed from the operands.  `leak` lets every
    row see one key more, as a mask off by one would: "limit" the key slot just past the row's last visible key (a
    zero-filled pad slot when that is Lk), "next_seq" the first key of the next sequence of the same packed tile (a pad
    slot for the tile's last sequence).  With QK-norm / RoPE on, "rope_shift" stages every row with the RoPE tables of
    the next position and "split" moves norm_split one token later (the first second-stream token gets the first pair)."""
    if leak in ("rope_shift", "split"):
        st = dict(case.stage)
        if leak == "split":
            st["split"] += 1
        else:
            st["cos"], st["sin"] = st["cos"].roll(-1, 0), st["sin"].roll(-1, 0)
        case, leak = copy.copy(case), None
        case.stage = st
    qu, ku, scl = _operands(case)
    v = case.v.double()
    out = torch.zeros(case.nseq, case.H, case.Lq, case.D, dtype=torch.float64, device=case.q.device)
    for s, r0, r1 in _chunks(case):
        S = scores(case, s, r0, r1, qu, ku, scl)[0]                             # [H, r, Lk]
        ex_s = torch.full(S.shape[:2], -math.inf, dtype=torch.float64, device=S.device)
        ex_v = torch.zeros(*S.shape[:2], case.D, dtype=torch.float64, device=S.device)
        if leak == "limit":
            lim = visible(case, s, s + 1, r0, r1)[0].expand(case.H, -1, -1).sum(-1)   # [H, r]: a prefix of keys
            k_ = lim.clamp(max=case.Lk - 1)
            real = lim < case.Lk
            kk = ku[s][torch.arange(case.H, device=S.device)[:, None], k_]                  # [H, r, D]
            ex_s = torch.where(real, (qu[s, :, r0:r1] * kk).sum(-1) * scl, 0.0)
            ex_v = torch.where(real[..., None], v[s][torch.arange(case.H, device=S.device)[:, None], k_], 0.0)
        elif leak == "next_seq":
            if s + 1 < case.nseq and s // case.pack == (s + 1) // case.pack:
                ex_s = (qu[s, :, r0:r1] * ku[s + 1, :, :1]).sum(-1) * scl
                ex_v = v[s + 1, :, :1].expand(-1, r1 - r0, -1)
            else:
                ex_s = torch.zeros_like(ex_s)
        m = torch.maximum(S.amax(-1), ex_s)
        live = m > -math.inf
        m = torch.where(live, m, 0.0)
        p = torch.exp2(S - m[..., None])
        pe = torch.exp2(ex_s - m)
        num = p @ v[s] + pe[..., None] * ex_v
        den = p.sum(-1) + pe
        out[s, :, r0:r1] = torch.where(live[..., None], num / den.clamp(min=1e-300)[..., None], 0.0)
    return out


# ---- operands ---------------------------------------------------------------------------------------------------------
def _values(g, nseq, H, Lk, D, tie_keys):
    """Values [nseq, H, Lk, D] (see the module docstring); tie_keys: list of (seq, LongTensor of tied keys)."""
    dev = g.device
    nb = -(-Lk // 128)
    # E_max per (sequence, head, channel) in [-3, 1], reached by one 128-key block; the other blocks 0 to 2 below it
    emax = _randint(g, 5, (nseq, H, 1, D)) - 3
    Eb = emax - _randint(g, 3, (nseq, H, nb, D))
    top = _randint(g, nb, (nseq, H, 1, D))
    Eb = torch.where(torch.arange(nb, device=dev)[:, None] == top, emax, Eb)
    E = Eb.repeat_interleave(128, 2)[:, :, :Lk]
    e = E - _randint(g, 4, (nseq, H, Lk, D))
    m = 1.0 + 0.25 * _randint(g, 4, (nseq, H, Lk, D)).float()
    sign = 1.0 - 2.0 * _randint(g, 2, (nseq, H, Lk, D)).float()
    v = sign * torch.ldexp(m, e)
    tied = torch.zeros(nseq, Lk, dtype=torch.bool, device=dev)
    for s, keys in tie_keys:      # tied winners: one exponent per channel (the lowest E of their groups)
        emin = E[s][:, keys].amin(1, keepdim=True)                            # [H, 1, D]
        v[s][:, keys] = sign[s][:, keys] * torch.ldexp(m[s][:, keys], emin.expand(-1, len(keys), -1))
        tied[s, keys] = True
    # plant +-1.75 x 2^E in every (sequence, head, 128-key block, channel) on a key that is not a tied winner
    pick = torch.rand(nseq, H, Lk, D, generator=g, device=dev) - 2.0 * tied[:, None, :, None]
    pick = torch.nn.functional.pad(pick, (0, 0, 0, nb * 128 - Lk), value=-9.0).view(nseq, H, nb, 128, D)
    best = pick.argmax(3)                                                     # [nseq, H, nb, D]
    if bool((pick.amax(3) < 0).any()):
        raise BudgetError("a 128-key block holds only tied winners: no key left for its value scale")
    key = best + 128 * torch.arange(nb, device=dev)[:, None]
    idx = (torch.arange(nseq, device=dev)[:, None, None, None], torch.arange(H, device=dev)[None, :, None, None],
           key, torch.arange(D, device=dev))
    v[idx] = sign[idx] * torch.ldexp(torch.full_like(m[idx], 1.75), E[idx])
    return v


def _design(g, nseq, H, Lq, Lk, D, grp, cand, cnt, decoys, negative=True, dups=()):
    """q [nseq, H, Lq, D] (alpha x units), k [nseq, H, Lk, D], decoy pairs [nd, 4] and tied key lists.
    grp [Lq]: row group of every query row; cand [nseq, ngr, W, t]: the winner units (t tied keys each) of every group,
    the first cnt[s, group] valid; decoys [(seq_q, group, seq_k, key0, n)]: keys key0 + u of seq_k get twice the code of
    unit u of the group, for u < min(n, cnt) (rows picking unit u then have a decoy there); dups [(seq, group, key0, n)]:
    keys key0 + u get the code of unit u at the same magnitude (visible copies, for cases whose streams scale keys
    differently)."""
    dev = g.device
    NC = n_codes(D)
    gs = (D - 1) // 3
    W, t = cand.shape[2], cand.shape[3]
    valid = torch.arange(W, device=dev) < cnt[..., None]                      # [nseq, ngr, W]
    seq_of = torch.arange(nseq, device=dev)[:, None, None].expand_as(valid)
    firsts = cand[..., 0]
    uniq, inv = torch.unique(seq_of[valid] * Lk + firsts[valid], return_inverse=True)
    U = len(uniq)
    if U > NC - FILLERS:
        raise BudgetError(f"{U} winner units need more than the {NC - FILLERS} codes of head_dim {D}")
    unit_of = torch.full((nseq * Lk,), -1, dtype=torch.long, device=dev)
    unit_of[uniq] = torch.arange(U, device=dev)
    ids = torch.stack([torch.randperm(NC - FILLERS, generator=g, device=dev)[:U] for _ in range(H)])     # [H, U]
    codes = (NC - FILLERS) + _randint(g, FILLERS, (H, nseq, Lk))
    kmul = torch.ones(nseq, Lk, device=dev)
    flat_s = seq_of[valid]
    tie_keys = []
    for j in range(t):
        keys = cand[..., j][valid]
        codes[:, flat_s, keys] = ids[:, inv]
    if t > 1:
        for s in range(nseq):
            sel = cand[s][valid[s]]                                           # [units, t]
            for row in torch.unique(sel, dim=0):
                tie_keys.append((s, row))
    # rows: a unit of their group
    unit_idx = _randint(g, cnt[:, grp].clamp(min=1), (nseq, Lq))                         # [nseq, Lq]
    win_first = cand[torch.arange(nseq, device=dev)[:, None], grp[None], unit_idx, 0]   # [nseq, Lq]
    has = cnt[:, grp] > 0
    row_unit = unit_of[(torch.arange(nseq, device=dev)[:, None] * Lk + win_first).clamp(min=0)]
    row_codes = torch.where(has[None], ids[:, row_unit.clamp(min=0)], (NC - FILLERS) + _randint(g, FILLERS, (H, nseq, Lq)))
    pairs = []
    for sq, gr, sk, key0, nmax in decoys:
        n = min(int(cnt[sq, gr]), Lk - key0, nmax)
        for u in range(n):
            ufirst = int(cand[sq, gr, u, 0])
            codes[:, sk, key0 + u] = ids[:, int(unit_of[sq * Lk + ufirst])]
            kmul[sk, key0 + u] = 2.0
            rows = ((grp == gr) & (unit_idx[sq] == u)).nonzero().flatten()
            if len(rows):
                pairs.append(torch.stack([torch.full_like(rows, sq), rows, torch.full_like(rows, sk),
                                          torch.full_like(rows, key0 + u)], 1))
    for s_, gr, key0, nmax in dups:
        for u in range(min(int(cnt[s_, gr]), nmax)):
            codes[:, s_, key0 + u] = ids[:, int(unit_of[s_ * Lk + int(cand[s_, gr, u, 0])])]
    k = code_vectors(codes, D) * kmul[None, :, :, None]
    k[..., 3 * gs] = 1.0
    q = code_vectors(row_codes, D)
    if negative:
        q[..., 3 * gs] = torch.where(_randint(g, 2, (H, nseq, Lq)) == 1, NEG, 0.0)
    q = q * ALPHA[D]
    dpairs = torch.cat(pairs) if pairs else torch.zeros(0, 4, dtype=torch.long, device=dev)
    return q.transpose(0, 1).contiguous(), k.transpose(0, 1).contiguous(), dpairs, tie_keys


def _cand_range(g, lo, hi, W, t=1):
    """[W', t] winner units in keys [lo, hi): the first, the middle and the last key plus random others (t == 1), or W'
    tuples of t keys (hi - lo) / t apart (ties across key blocks).  W' = min(W, number possible)."""
    n = hi - lo
    if n <= 0:
        return torch.zeros(0, t, dtype=torch.long, device=g.device)
    if t == 1:
        fixed = torch.tensor(sorted({lo, lo + n // 2, hi - 1}), device=g.device)
        rest = lo + torch.randperm(n, generator=g, device=g.device)
        keys = torch.cat([fixed, rest[~torch.isin(rest, fixed)]])[:min(W, n)]
        return keys[:, None]
    step = n // t
    base = lo + torch.randperm(step, generator=g, device=g.device)[:min(W, step // 4)]   # most keys stay untied
    return base[:, None] + step * torch.arange(t, device=g.device)


def _stack_cands(lists, W, t, dev):
    """lists[s][gr] -> (cand [nseq, ngr, W, t], cnt [nseq, ngr])."""
    nseq, ngr = len(lists), len(lists[0])
    cand = torch.zeros(nseq, ngr, W, t, dtype=torch.long, device=dev)
    cnt = torch.zeros(nseq, ngr, dtype=torch.long, device=dev)
    for s in range(nseq):
        for gr in range(ngr):
            c = lists[s][gr]
            cand[s, gr, :len(c)] = c
            cnt[s, gr] = len(c)
    return cand, cnt


class AttnCase:
    """One call with exact operands, designed per sequence: q [nseq, H, Lq, D], k / v [nseq, H, Lk, D] (bf16-exact
    fp32), the visibility inputs (kv_lens [nseq], bias [Hb, Lq + Lk - 1], frames (frame_tokens, q_frame0)), decoy pairs
    (seq_q, row, seq_k, key) and, after check_budget, the expected rows.  `run(impl)` lays the operands out for the entry
    point and calls it on `impl` (the binding or a CPU stand-in); `got(...)` / `want()` give output and expectation in
    the token layout, `untouched()` whether everything around the output view kept its sentinel."""

    pack = 1

    def __init__(self, name, q, k, v, *, scale=None, kv_lens=None, bias=None, frames=None, decoys=None, tie_keys=(),
                 stage=None):
        self.name = name
        self.q, self.k, self.v = q, k, v
        self.nseq, self.H, self.Lq, self.D = q.shape
        self.Lk = k.shape[2]
        self.alpha = ALPHA[self.D]
        self.scale = scale if scale is not None else self.D ** -0.5
        self.kv_lens, self.bias, self.frames, self.decoys = kv_lens, bias, frames, decoys
        self.tie_keys, self.stage = tie_keys, stage
        check_budget(self)

    def __repr__(self):
        return self.name


def _gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def _bf(x):
    return x.to(torch.bfloat16)


def _sentinel_out(rows, cols, dev, dtype=torch.bfloat16, fill=SENTINEL):
    buf = torch.full((rows, cols + 2 * PAD), fill, dtype=torch.float32, device=dev).to(dtype)
    return buf, buf[:, PAD:PAD + cols]


def _untouched(buf, cols, fill):
    outside = torch.cat([buf[:, :PAD], buf[:, PAD + cols:]], 1)
    return bool((outside.float() == fill).all())


def _token_rows(x, rows):
    """[nseq, H, L, D] -> [R, H * D] with (seq, pos) at token row rows[seq, pos]."""
    nseq, H, L, D = x.shape
    out = torch.zeros(int(rows.max()) + 1, H * D, dtype=x.dtype, device=x.device)
    out[rows.reshape(-1)] = x.permute(0, 2, 1, 3).reshape(nseq * L, H * D)
    return out


# ---- attn_tiles / attn_tiles_fp8 --------------------------------------------------------------------------------------
def _stream_rows(mode, B, T, S, nseq, L, dev):
    """[nseq, L] token row of (sequence, position) in a [B, T, S] frame-major stream: mode 0 sequences along S, mode 1
    along T."""
    s = torch.arange(nseq, device=dev)[:, None]
    p = torch.arange(L, device=dev)[None]
    if mode == 0:
        return s * L + p
    return ((s // S) * T + p) * S + s % S


class TilesSelfCase(AttnCase):
    def run(self, impl):
        import osb200 as real
        dev = self.q.device
        H, D, L = self.H, self.D, self.Lq
        tm = real.tile_map(0, self.L_seq) if self.mode == 0 else real.tile_map(1, self.T, self.S, self.T)
        out_map = None
        if self.transposed:
            tm, out_map = real.tile_map(0, self.T), tm
        x = torch.cat([_token_rows(_bf(t), self.in_rows) for t in (self.q, self.k, self.v)], 1)
        w = torch.eye(3 * H * D, dtype=torch.bfloat16, device=dev)
        tiles = impl.HeadTiles(x.shape[0], tm, 3, H, D, dev)
        impl.gemm_head_tiles(x, w, None, tiles, nkinds=3)
        self.buf, out = _sentinel_out(x.shape[0], H * D, dev)
        self.tmap = tm
        if self.fp8:
            t8 = impl.HeadTilesFp8(tiles)
            impl.head_tiles_fp8(tiles, t8, v_period=3, v_slot=2)
            impl.attn_tiles_fp8(t8, t8, out, Lk=L, num_seqs=self.nseq, out_map=out_map)
        elif self.scatter:   # osb_scatter mode 2 with one rank: rows [B, T, S] split along T over P = 1
            sc = impl.make_scatter(2, 1, 0, self.T, self.S, [out])
            impl.attn_tiles(tiles, tiles, None, Lk=L, num_seqs=self.nseq, out_map=out_map, out_scatter=sc,
                            out_ld=out.stride(0))
        else:
            impl.attn_tiles(tiles, tiles, out, Lk=L, num_seqs=self.nseq, out_map=out_map)
        return out

    def want(self):
        return _token_rows(self.expected, self.out_rows).to(torch.bfloat16)

    def untouched(self):
        return _untouched(self.buf, self.H * self.D, SENTINEL)


def tiles_self_case(mode, B, T, S, H, D, *, transposed=False, ties=1, fp8=False, scatter=False, W=8, seed=0,
                    device="cpu"):
    """Self-attention over head tiles written by `gemm_head_tiles` with W = I (the tiles hold the designed rows exactly):
    mode 0 spatial (sequences of S tokens), mode 1 temporal (sequences of T frames of a frame-major stream, packed
    128 // T per tile when T <= 64); `transposed`: tiles from the [B, S, T] stream, output rows frame-major (out_map);
    `scatter`: the output rows routed through osb_scatter mode 2 with one rank (bf16, temporal)."""
    import osb200 as real
    g = _gen(seed, device)
    L = S if mode == 0 else T
    nseq = B * T if mode == 0 else B * S
    tm = real.tile_map(0, S) if mode == 0 else real.tile_map(1, T, S, T)
    G = tm.G
    nd = min(W, L // 4) if G > 1 else 0          # decoy slots at the start of the next packed sequence
    lists = [[_cand_range(g, nd, L, W, ties)] for _ in range(nseq)]
    cand, cnt = _stack_cands(lists, W, ties, g.device)
    decoys = [(s, 0, s + 1, 0, nd) for s in range(nseq - 1) if G > 1 and s // G == (s + 1) // G]
    grp = torch.zeros(L, dtype=torch.long, device=g.device)
    q, k, dp, tk = _design(g, nseq, H, L, L, D, grp, cand, cnt, decoys)
    v = _values(g, nseq, H, L, D, tk)
    name = (f"attn_tiles{'_fp8' if fp8 else ''} {'spatial' if mode == 0 else 'temporal'} B={B} T={T} S={S} H={H} D={D}"
            + (" transposed" if transposed else "") + (" scatter" if scatter else "") + (f" ties={ties}" if ties > 1 else ""))
    c = TilesSelfCase(name, q, k, v, decoys=dp, tie_keys=tk)
    assert not scatter or (mode == 1 and not fp8)
    c.mode, c.B, c.T, c.S, c.L_seq, c.transposed, c.fp8, c.pack, c.G = mode, B, T, S, L, transposed, fp8, G, G
    c.scatter = scatter
    rows = _stream_rows(mode, B, T, S, nseq, L, g.device)
    c.out_rows = rows
    c.in_rows = (torch.arange(nseq, device=g.device)[:, None] * L + torch.arange(L, device=g.device)[None]
                 if transposed else rows)
    c.items = H * (-(-nseq // G) if G > 1 else nseq) * tm.tps
    return c


class TilesCrossCase(AttnCase):
    def run(self, impl):
        import osb200 as real
        dev = self.q.device
        H, D, B, N, Ly = self.H, self.D, self.nseq, self.Lq, self.Lk
        xq = _token_rows(_bf(self.q), self.q_rows)
        y = torch.cat([_token_rows(_bf(t), self.k_rows) for t in (self.k, self.v)], 1)
        qt = impl.HeadTiles(B * N, real.tile_map(0, N), 1, H, D, dev)
        kt = impl.HeadTiles(B * Ly, real.tile_map(0, Ly, keys_only=True), 2, H, D, dev)
        impl.gemm_head_tiles(xq, torch.eye(H * D, dtype=torch.bfloat16, device=dev), None, qt, nkinds=1)
        impl.gemm_head_tiles(y, torch.eye(2 * H * D, dtype=torch.bfloat16, device=dev), None, kt, nkinds=2)
        self.buf, out = _sentinel_out(B * N, H * D, dev)
        lens = self.kv_lens.to(dev)
        if self.fp8:
            q8, k8 = impl.HeadTilesFp8(qt), impl.HeadTilesFp8(kt)
            impl.head_tiles_fp8(qt, q8)
            impl.head_tiles_fp8(kt, k8, v_period=2, v_slot=1)
            impl.attn_tiles_fp8(q8, k8, out, q_kind=0, k_kind=0, v_kind=1, Lk=Ly, num_seqs=B, kv_lens=lens)
        else:
            impl.attn_tiles(qt, kt, out, q_kind=0, k_kind=0, v_kind=1, Lk=Ly, num_seqs=B, kv_lens=lens)
        return out

    def want(self):
        return _token_rows(self.expected, self.q_rows).to(torch.bfloat16)

    def untouched(self):
        return _untouched(self.buf, self.H * self.D, SENTINEL)


def tiles_cross_case(N, Ly, lens, H, D, *, fp8=False, W=8, seed=0, device="cpu"):
    """Cross-attention over head tiles: len(lens) samples of N query tokens, Ly text keys each, the first lens[b] valid.
    Decoys fill the slots just past lens[b]; lens[b] == 0 rows must come out zero."""
    g = _gen(seed, device)
    B = len(lens)
    lists = [[_cand_range(g, 0, n, W)] for n in lens]
    cand, cnt = _stack_cands(lists, W, 1, g.device)
    decoys = [(b, 0, b, n, W) for b, n in enumerate(lens) if 0 < n < Ly]
    grp = torch.zeros(N, dtype=torch.long, device=g.device)
    q, k, dp, tk = _design(g, B, H, N, Ly, D, grp, cand, cnt, decoys)
    v = _values(g, B, H, Ly, D, tk)
    kv_lens = torch.tensor(lens, dtype=torch.int32, device=g.device)
    name = f"attn_tiles{'_fp8' if fp8 else ''} cross N={N} Ly={Ly} lens={list(lens)} H={H} D={D}"
    c = TilesCrossCase(name, q, k, v, kv_lens=kv_lens, decoys=dp)
    c.fp8 = fp8
    c.q_rows = torch.arange(B * N, device=g.device).view(B, N)
    c.k_rows = torch.arange(B * Ly, device=g.device).view(B, Ly)
    c.items = H * B * -(-N // 128)
    return c


# ---- attn_short / attn_fp8 / attn_fp8_blocks --------------------------------------------------------------------------
class ShortCase(AttnCase):
    """Token-layout q / k / v as column slices of one [rows, 3 H D + 16] buffer; output a column slice of a sentinel
    buffer.  `seqs_per_batch` > 1: short sequences, `seqs_per_batch` of them per batch element."""
    fn = "attn_short"

    def _operands(self):
        dev = self.q.device
        HD = self.H * self.D
        rows = self.nseq * max(self.Lq, self.Lk)
        buf = torch.zeros(rows, 3 * HD + 16, dtype=torch.bfloat16, device=dev)
        k_rows = torch.arange(self.nseq * self.Lk, device=dev).view(self.nseq, self.Lk)
        for i, (t, r) in enumerate(((self.q, self.rows), (self.k, k_rows), (self.v, k_rows))):
            x = _token_rows(_bf(t), r)
            buf[:x.shape[0], i * HD:(i + 1) * HD] = x
        L, spb = self.Lq, self.spb
        kw = dict(num_seqs=self.nseq, seqs_per_batch=spb, q_strides=(spb * L, L, 1),
                  k_strides=(spb * self.Lk, self.Lk, 1), Lq=L, Lk=self.Lk,
                  num_heads=self.H, head_dim=self.D)
        if self.kv_lens is not None:
            kw["kv_lens"] = self.kv_lens
        if self.scale != self.D ** -0.5:
            kw["softmax_scale"] = self.scale
        if self.stage is not None:
            st = self.stage
            kw.update(q_norm_w=st["qw"], k_norm_w=st["kw"], q_norm_w2=st["qw2"], k_norm_w2=st["kw2"],
                      norm_split=st["split"], norm_eps=st["eps"], rope_cos=st["cos"], rope_sin=st["sin"],
                      rope_half=st["half"])
        return buf[:, :HD], buf[:, HD:2 * HD], buf[:, 2 * HD:3 * HD], kw

    def run(self, impl):
        q, k, v, kw = self._operands()
        dev = q.device
        HD = self.H * self.D
        if self.fn == "attn_fp8_blocks":
            self.buf = torch.full((self.nseq * self.Lq, HD + 2 * 16), 0x5A, dtype=torch.uint8, device=dev)
            self.sbuf = torch.full((self.nseq * self.Lq, self.H + 2), SENTINEL, dtype=torch.float32, device=dev)
            out, out_s = self.buf[:, 16:16 + HD].view(E4M3), self.sbuf[:, 1:1 + self.H]
            ws = impl.attn_fp8_workspace(self.nseq, self.Lq, self.H, dev)
            return impl.attn_fp8_blocks(q, k, v, out, out_s, workspace=ws, **kw)
        self.buf, out = _sentinel_out(self.nseq * self.Lq, HD, dev)
        if self.fn == "attn_fp8":
            ws = impl.attn_fp8_workspace(self.nseq, self.Lq, self.H, dev)
            return impl.attn_fp8(q, k, v, out, workspace=ws, **kw)
        if self.fn == "attn_short_bias":
            kw.pop("softmax_scale", None)
            return impl.attn_short_bias(q, k, v, out, self.bias, softmax_scale=self.scale, **kw)
        return impl.attn_short(q, k, v, out, **kw)

    def want(self):
        w = _token_rows(self.expected, self.rows)
        if self.fn != "attn_fp8_blocks":
            return w.to(torch.bfloat16)
        # the block rule applied to the exact rows: s = amax / 448 per (row, head) (1 for a zero block), e4m3(v / s)
        x = w.float().view(w.shape[0], self.H, self.D)
        amax = x.abs().amax(-1)
        s = torch.where(amax > 0, amax / torch.full_like(amax, 448.0), torch.ones_like(amax))
        return (x / s[..., None]).clamp(-448.0, 448.0).to(E4M3).view(w.shape[0], -1), s

    def untouched(self):
        if self.fn == "attn_fp8_blocks":
            HD = self.H * self.D
            ok_c = bool((torch.cat([self.buf[:, :16], self.buf[:, 16 + HD:]], 1) == 0x5A).all())
            ok_s = bool((torch.cat([self.sbuf[:, :1], self.sbuf[:, 1 + self.H:]], 1) == SENTINEL).all())
            return ok_c and ok_s
        return _untouched(self.buf, self.H * self.D, SENTINEL)


# constant RMSNorm weights (q, k) of the first stream, per head_dim: one unit of code overlap scores ~70 log2 units
NORM_W = {64: (4.0, 5.25), 72: (4.0, 5.0), 128: (4.0, 3.75)}


def _stage_args(g, L, D, split, rope):
    """QK-norm weights (the second stream at twice the first) and quarter-turn RoPE tables [L, D/2] for short_case."""
    dev = g.device
    wq, wk = NORM_W[D]
    full = lambda x: torch.full((D,), x, dtype=torch.bfloat16, device=dev)   # noqa: E731
    turn = _randint(g, 4, (L, D // 2))
    cos = torch.tensor([1.0, 0.0, -1.0, 0.0], device=dev)[turn].contiguous()
    sin = torch.tensor([0.0, 1.0, 0.0, -1.0], device=dev)[turn].contiguous()
    return dict(qw=full(wq), kw=full(wk), qw2=full(2 * wq), kw2=full(2 * wk), split=split, eps=1e-6, cos=cos, sin=sin,
                half=rope == "half")


def short_case(L, H, D, *, B=1, T=1, kv_lens=None, ties=1, fn="attn_short", norm_split=None, rope=None, W=64, seed=0,
               device="cpu"):
    """`attn_short` (or `attn_fp8` / `attn_fp8_blocks` with D = 128): B batch elements of T sequences of L tokens,
    optional kv_lens [B T] with decoys just past each.  Sequences shorter than 128 tokens share a query tile 128 // L at a
    time, across batch elements: decoys sit at the first keys of the next sequence of the same tile.
    `norm_split` / `rope` ("interleaved" or "half"): QK-norm with two weight pairs split at norm_split and quarter-turn
    RoPE (see the module docstring); winners in [norm_split, L), each with a half-score copy among the first keys."""
    g = _gen(seed, device)
    nseq = B * T
    lens = list(kv_lens) if kv_lens is not None else [L] * nseq
    G = 128 // L if L < 128 else 1
    nd = min(8, L // 4) if G > 1 else 0
    host = [G > 1 and n > nd for n in lens]      # sequences whose first nd keys hold the previous sequence's decoys
    stage = None
    if norm_split is not None:
        assert kv_lens is None and G == 1 and ties == 1 and 0 < norm_split < L
        W = min(W, norm_split, L - norm_split)
        lists = [[_cand_range(g, norm_split, L, W)] for _ in range(nseq)]
    else:
        lists = [[_cand_range(g, nd if host[s] else 0, n, W, ties)] for s, n in enumerate(lens)]
    cand, cnt = _stack_cands(lists, W, ties, g.device)
    decoys = [(s, 0, s, n, W) for s, n in enumerate(lens) if n < L and cnt[s, 0] > 0]
    decoys += [(s, 0, s + 1, 0, nd) for s in range(nseq - 1) if s // G == (s + 1) // G and host[s + 1] and cnt[s, 0] > 0]
    dups = [(s, 0, 0, W) for s in range(nseq)] if norm_split is not None else ()
    grp = torch.zeros(L, dtype=torch.long, device=g.device)
    q, k, dp, tk = _design(g, nseq, H, L, L, D, grp, cand, cnt, decoys, negative=norm_split is None, dups=dups)
    if norm_split is not None:
        stage = _stage_args(g, L, D, norm_split, rope)
        if rope is not None:      # operands in pre-RoPE space: the kernel's RoPE brings them to the designed rows
            q = rope_rows(q.double(), stage["cos"], stage["sin"], stage["half"], inverse=True).float()
            k = rope_rows(k.double(), stage["cos"], stage["sin"], stage["half"], inverse=True).float()
        else:
            stage["cos"] = stage["sin"] = None
    v = _values(g, nseq, H, L, D, tk)
    kvl = torch.tensor(kv_lens, dtype=torch.int32, device=g.device) if kv_lens is not None else None
    name = f"{fn} L={L} B={B} T={T} H={H} D={D}" + (f" kv_lens={list(kv_lens)}" if kv_lens is not None else "") + (
        f" ties={ties}" if ties > 1 else "") + (f" norm_split={norm_split} rope={rope}" if norm_split is not None else "")
    c = ShortCase(name, q, k, v, kv_lens=kvl, decoys=dp, tie_keys=tk, stage=stage)
    c.fn, c.spb, c.pack = fn, T, G
    c.rows = torch.arange(nseq * L, device=g.device).view(nseq, L)
    return c


def t5_bias_case(Lq, Lk, H, *, B=2, variant="inf", seed=0, device="cpu"):
    """`attn_short_bias` with q = 0, so every score is the bias: head h's winner is the key at relative offset d_h
    (0 <= d_h <= Lk - Lq, in range for every row).  variant "inf": every other offset -inf (key blocks skipped);
    "finite": -300 (the same bits); "empty": head 0's only finite offset is Lk - 1, which only row 0 reaches, so every
    other row of head 0 sees no key and must come out zero."""
    g = _gen(seed, device)
    D = 64
    d = _randint(g, Lk - Lq + 1, (H,))
    # heads 1 and 2 on the edges of the key-block skip test of a 128-row query tile: offset 1 is the first live relative
    # position of key block k0 = 128 for rows 0..127, offset 63 the last of key block 0 (64 keys)
    d[1:3] = torch.tensor([1, min(63, Lk - Lq)], device=g.device)[:max(0, min(2, H - 1))]
    n = Lq + Lk - 1
    bias = torch.full((H, n), -math.inf if variant != "finite" else -300.0, device=g.device)
    bias[torch.arange(H, device=g.device), d + Lq - 1] = 0.0
    if variant == "empty":
        bias[0] = -math.inf
        bias[0, Lk - 1 + Lq - 1] = 0.0
    q = torch.zeros(B, H, Lq, D, device=g.device)
    codes = _randint(g, n_codes(D), (B, H, Lk))
    k = code_vectors(codes, D)
    v = _values(g, B, H, Lk, D, [])
    c = ShortCase(f"attn_short_bias t5 Lq={Lq} Lk={Lk} H={H} B={B} {variant}", q, k, v, scale=1.0, bias=bias.contiguous())
    c.fn, c.spb = "attn_short_bias", 1
    c.rows = torch.arange(B * Lq, device=g.device).view(B, Lq)
    c.offsets = d
    return c


def causal_case(L, H, *, B=1, seed=0, device="cpu"):
    """`attn_short_bias` with CLIP's causal mask (one shared bias: 0 for j <= i, -inf for j > i).  Rows i = 7 mod 8 win
    on their own key i and have a decoy at j = i + 1 (twice their code); every other row wins on a random earlier key
    that is neither such a key nor a decoy."""
    g = _gen(seed, device)
    D = 64
    own = [i for i in range(L) if i % 8 == 7]
    taken = set(own) | {i + 1 for i in own}
    lists = []
    for s in range(B):
        per = []
        for i in range(L):
            if i % 8 == 7:
                per.append(torch.tensor([[i]], device=g.device))
            else:
                free = torch.tensor([j for j in range(i + 1) if j not in taken], device=g.device)
                per.append(free[torch.randperm(len(free), generator=g, device=g.device)[:8]][:, None])
        lists.append(per)
    cand, cnt = _stack_cands(lists, 8, 1, g.device)
    grp = torch.arange(L, device=g.device)
    decoys = [(s, i, s, i + 1, 1) for s in range(B) for i in own if i + 1 < L]
    q, k, dp, tk = _design(g, B, H, L, L, D, grp, cand, cnt, decoys)
    v = _values(g, B, H, L, D, tk)
    n = 2 * L - 1
    bias = torch.where(torch.arange(n, device=g.device) <= L - 1, 0.0, -math.inf)
    c = ShortCase(f"attn_short_bias causal L={L} H={H} B={B}", q, k, v, bias=bias.contiguous(), decoys=dp)
    c.fn, c.spb = "attn_short_bias", 1
    c.rows = torch.arange(B * L, device=g.device).view(B, L)
    return c


# ---- attn_frames ------------------------------------------------------------------------------------------------------
class FramesCase(AttnCase):
    """q [batch, Lq, 512], k / v [batch, Lk, 512] as column slices of wider buffers (k | v side by side); out a column
    slice of a sentinel buffer."""

    def run(self, impl):
        dev = self.q.device
        nb, Lq, Lk, D = self.nseq, self.Lq, self.Lk, self.D
        qb = torch.zeros(nb, Lq, D + 16, dtype=torch.bfloat16, device=dev)
        qb[..., 8:8 + D] = _bf(self.q[:, 0])
        kvb = torch.zeros(nb, Lk, 2 * D + 16, dtype=torch.bfloat16, device=dev)
        kvb[..., :D] = _bf(self.k[:, 0])
        kvb[..., D:2 * D] = _bf(self.v[:, 0])
        self.buf = torch.full((nb, Lq, D + 2 * PAD), SENTINEL, dtype=torch.bfloat16, device=dev)
        out = self.buf[..., PAD:PAD + D]
        hw, f0 = self.frames
        impl.attn_frames(qb[..., 8:8 + D], kvb[..., :D], kvb[..., D:2 * D], frame_tokens=hw, q_frame0=f0, out=out)
        return out

    def want(self):
        return self.expected[:, 0].to(torch.bfloat16)

    def untouched(self):
        return bool((torch.cat([self.buf[..., :PAD], self.buf[..., PAD + self.D:]], -1).float() == SENTINEL).all())


def frames_case(hw, q_frames, *, q_frame0=0, k_frames=None, batch=1, W=8, seed=0, device="cpu"):
    """`attn_frames`: queries are frames q_frame0 .. q_frame0 + q_frames - 1 of a video of k_frames frames of hw tokens.
    A row of frame F wins on a key of frame F (the row's last visible key block), away from the first W slots of the
    frame, which hold the decoys of frame F - 1's winners."""
    g = _gen(seed, device)
    D = 512
    k_frames = k_frames if k_frames is not None else q_frame0 + q_frames
    Lq, Lk = q_frames * hw, k_frames * hw
    nd = min(W, hw // 2)
    lists = [[_cand_range(g, F * hw + nd, (F + 1) * hw, W) for F in range(q_frame0, q_frame0 + q_frames)]
             for _ in range(batch)]
    cand, cnt = _stack_cands(lists, W, 1, g.device)
    grp = torch.arange(Lq, device=g.device) // hw
    decoys = [(b, f, b, (q_frame0 + f + 1) * hw, nd) for b in range(batch) for f in range(q_frames)
              if (q_frame0 + f + 1) * hw < Lk]
    q, k, dp, tk = _design(g, batch, 1, Lq, Lk, D, grp, cand, cnt, decoys)
    v = _values(g, batch, 1, Lk, D, tk)
    name = f"attn_frames hw={hw} frames {q_frame0}..{q_frame0 + q_frames - 1} of {k_frames} batch={batch}"
    return FramesCase(name, q, k, v, frames=(hw, q_frame0), decoys=dp)
