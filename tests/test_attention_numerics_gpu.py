"""Attention kernels against an fp64 reference, with the attention mass placed where a kernel can go wrong.

Unit-randn q / k / v give a nearly flat softmax: every output is an average of hundreds of random V rows, of size ~1/sqrt(n),
and a blanket 2e-2 tolerance is half of that signal. A kernel that drops the new token, shifts a causal mask by one or loses a
split passes such a test. Here every case builds inputs whose mass sits on the keys at the edges (a tile's last key, a split's
last key, the diagonal, the new token, seq_len - 1) and puts finite "poison" (a key aimed at the query with V = +-1e3) on the
keys a kernel must not attend. The bound per output element is

    |got - ref| <= KAPPA * (2^-8 * sum_j p_j |v_j| + 2^-8 * |ref|)

The first term covers P rounded to bf16 before the PV product (the flash kernels; the mq kernel's hi + lo split is tighter),
the second the bf16 output. It scales with sum p|v|, not |ref|, so cancellation in the output does not blow it up.

test_mutated_references_violate_the_bound (CPU) shows the inputs are sharp: for every case it computes plausible wrong answers
(a needle or the new token dropped, the mask shifted by one either way, a split's key range dropped, `scale` in place of
`scale * log2(e)` in the exponent, one poisoned key attended) and asserts each one falls outside the bound. The GPU tests run
the same cases through the kernels. The decode kernels rope q and the new k themselves; the reference attends with the rows
b2_op_rope_kv_write_at produces (the same device RoPE), and the RoPE tests at the end pin those rows to HF's within one bf16 ulp
(plus the angle difference of the two inv_freq formulas) and the prefill and decode cache rows to each other bit for bit. The
decode kernels' own RoPE of q is covered only indirectly: its table is the one pinned to HF, and a q roped differently would
move the needles' scores, which are 10+ above the rest, and show up in the attention bound.

The megakernel's attention phase has no op entry: the model-level tests run it, and every other decode path, on weights that
put each head's mass on the query's own key, which in a decode step is the new token."""
import math
import os
import subprocess
import sys

import pytest
import torch

from oracle import kv_fp8_oracle as KV
from oracle import llava_oracle as O

KAPPA = 4.0
ULP = 2.0 ** -8
T_NEEDLE = 16.0            # a needle's score, natural-log units (23 in the kernels' log2 units: far inside fp32 exp2)
NEEDLE_V, POISON_V, OFFSET_V = 8.0, 1e3, 30.0
DEV, BF = "cuda", torch.bfloat16
F64 = torch.float64


# ------------------------------------------------------------------------------------------------------ reference
def attend(pr, lim=None, scale=None, drop=(), extra=()):
    """fp64 attention of one (sample, head) problem: q [Q, D], k / v [N, D] (the bf16 values the kernel reads, as fp64); row i
    attends keys 0 .. lim[i]. Returns (out [Q, D], p [Q, N])."""
    q, k, v = pr["q"], pr["k"], pr["v"]
    lim = pr["lim"] if lim is None else lim
    s = (q @ k.T) * (pr["scale"] if scale is None else scale)
    allowed = torch.arange(k.shape[0])[None, :] <= lim[:, None]
    for r, key in extra:
        allowed[r, key] = True
    if len(drop):
        allowed[:, list(drop)] = False
    p = torch.softmax(s.masked_fill(~allowed, -math.inf), -1).nan_to_num(0.0)  # nothing attended -> 0
    return p @ v, p


def bound(pr, ref, p):
    return KAPPA * (ULP * (p @ pr["v"].abs()) + ULP * ref.abs())


def worst_ratio(pr, got, ref, p):
    rows = pr["rows"]
    return float(((got[rows] - ref[rows]).abs() / bound(pr, ref, p)[rows]).max())


def mutations(pr):
    """Plausible wrong answers of a kernel on this problem, as arguments of attend()."""
    out = {}
    for j in pr["needles"]:
        out[f"drop key {j}"] = dict(drop=[j])
    for b, e in pr.get("splits", ()):
        if e > b:
            out[f"drop split [{b}, {e})"] = dict(drop=range(b, e))
    lim, N = pr["lim"], pr["k"].shape[0]
    if bool((lim[pr["rows"]] + 1 < N).any()):
        out["mask +1"] = dict(lim=(lim + 1).clamp(max=N - 1))
    out["mask -1"] = dict(lim=lim - 1)
    out["scale without log2(e)"] = dict(scale=pr["scale"] * math.log(2.0))
    if pr["poison"]:
        out[f"attend poison {pr['poison'][0]}"] = dict(extra=[pr["poison"][0]])
    return out


# ------------------------------------------------------------------------------------------------------ input builder
def _aim_dir(q, scale):
    """Key direction that gives row q the score 1: q / (scale |q|^2)."""
    return q / (scale * (q * q).sum(-1, keepdim=True))


def _needle_v(g, key, D, bump=NEEDLE_V):
    v = 0.5 * torch.randn(D, generator=g, dtype=F64)
    v[(key * 37) % D] += bump
    return v


def _poison_v(g, D):
    return POISON_V * (torch.randint(0, 2, (D,), generator=g) * 2 - 1).to(F64)


def _place(g, q, k, v, aims, poison_keys, needle_keys, scale, D, bump):
    """Write the aimed keys into k / v (fp64, in place). aims: (key, row, score) triples. Keys aimed at a row that must not
    see them get poison V; other aimed keys a distinctive needle V."""
    touched = {}
    for key, row, t in aims:  # the first aim of a (key, row) pair wins: adding two would double the score
        if 0 <= key < k.shape[0] and row not in dict(touched.get(key, [])):
            touched.setdefault(key, []).append((row, t))
    for key, lst in touched.items():
        k[key] = sum(t * _aim_dir(q[row], scale) for row, t in lst)
        v[key] = _poison_v(g, D) if key in poison_keys else _needle_v(g, key, D, bump)
    return sorted(j for j in needle_keys if j in touched)


def _diag_aims(qpos, rows):
    """Per query row r at position qpos[r]: its own key (score T), the next key (score T: poison, r must not see it) and the
    previous key (T - 1.5, so a row weighs two keys and an error in the exponent scale shows)."""
    aims, poison = [], []
    for r in rows:
        p = int(qpos[r])
        aims += [(p, r, T_NEEDLE), (p + 1, r, T_NEEDLE), (p - 1, r, T_NEEDLE - 1.5)]
        poison.append((r, p + 1))
    return aims, poison


def _finish(g, q, k, v, lim, rows, scale, aims, poison, needles, regime, splits=()):
    D = q.shape[1]
    # a key no checked row may attend carries V = +-1e3; one that is another row's own key keeps a needle V, so the rows that
    # attend it are not swamped by it
    pkeys = {key for _, key in poison if key > int(lim[rows].max())}
    if regime == "flat":
        aims, poison, needles, pkeys = [], [], [], set()
    # on top of V = 30 + randn a needle's one-hot must still stand out against the 2^-8 * 30 part of the bound
    needles = _place(g, q, k, v, aims, pkeys, needles, scale, D, 10 * NEEDLE_V if regime == "offset" else NEEDLE_V)
    if regime == "offset":
        v += OFFSET_V
    return dict(q=q, k=k, v=v, lim=lim, rows=rows, scale=scale, needles=needles, splits=list(splits),
                poison=[(r, key) for r, key in poison if 0 <= key < k.shape[0] and key > lim[r]])


def bf(x):
    return x.to(BF).to(F64)


# ---- flash_attn (ViT / prefill from position 0) ----
def build_flash(c, seed):
    """q / k / v [B, S, H, D] bf16 and the problems [(b, h, problem)]."""
    B, S, H, D, causal = c["B"], c["S"], c["H"], c["D"], c["causal"]
    lens = c["lens"] or [S] * B
    g = torch.Generator().manual_seed(seed)
    scale = D ** -0.5
    q = bf(torch.randn(B, S, H, D, generator=g, dtype=F64))
    k = torch.randn(B, S, H, D, generator=g, dtype=F64)
    v = torch.randn(B, S, H, D, generator=g, dtype=F64)
    probs = []
    for b in range(B):
        n = lens[b]
        rows = torch.zeros(S, dtype=torch.bool)
        rows[:n] = True
        qpos = torch.arange(S)
        lim = qpos.clamp(max=n - 1) if causal else torch.full((S,), n - 1)
        edge = {0, 63, 64, 127, 128, n - 1}
        for h in range(H):
            kk, vv = k[b, :, h].clone(), v[b, :, h].clone()
            if causal:
                aims, poison = _diag_aims(qpos, range(n))
            else:
                targets = sorted({0, n // 2, n - 1})
                keys = sorted(j for j in edge if j < n)
                aims = [(j, r, T_NEEDLE - ((a + i) % 3)) for a, j in enumerate(keys) for i, r in enumerate(targets)]
                poison = [(r, j) for j in range(n, min(n + 2, S)) for r in targets]
                aims += [(j, r, T_NEEDLE + 2) for r, j in poison]
            pr = _finish(g, q[b, :, h], kk, vv, lim, rows, scale, aims, poison, edge, c["regime"])
            pr["k"], pr["v"] = bf(pr["k"]), bf(pr["v"])
            k[b, :, h], v[b, :, h] = pr["k"], pr["v"]
            probs.append((b, h, pr))
    return dict(q=q.to(BF), k=k.to(BF), v=v.to(BF), lens=c["lens"]), probs


# ---- flash_attn_kv (a prefill chunk at cache offset pos0) ----
def build_flash_kv(c, seed):
    """q [B, S, H, 128], caches [B, H, Smax, 128], pos0 / lens [B]."""
    B, S, H, D, Smax = len(c["pos0"]), c["S"], c["H"], 128, c["Smax"]
    g = torch.Generator().manual_seed(seed)
    scale = D ** -0.5
    q = bf(torch.randn(B, S, H, D, generator=g, dtype=F64))
    kc = torch.randn(B, H, Smax, D, generator=g, dtype=F64)
    vc = torch.randn(B, H, Smax, D, generator=g, dtype=F64)
    probs = []
    for b in range(B):
        p0, n = c["pos0"][b], c["lens"][b]
        rows = torch.zeros(S, dtype=torch.bool)
        rows[:n] = True
        qpos = p0 + torch.arange(S)
        lim = qpos.clamp(max=p0 + n - 1)
        for h in range(H):
            aims, poison = _diag_aims(qpos, range(n))
            prefix = sorted({0, p0 // 2, p0 - 1} - {-1}) if p0 > 0 else []
            aims += [(j, r, T_NEEDLE - 1 - (a % 2)) for a, j in enumerate(prefix) for r in sorted({0, n - 1})]
            poison += [(n - 1, j) for j in range(p0 + n + 1, min(p0 + n + 3, Smax))]
            aims += [(j, r, T_NEEDLE + 2) for r, j in poison[-2:] if j > p0 + n]
            needles = set(prefix) | {p0, p0 + n - 1, int(qpos[0]) + 63}
            pr = _finish(g, q[b, :, h], kc[b, h].clone(), vc[b, h].clone(), lim, rows, scale, aims, poison, needles,
                         c["regime"])
            pr["k"], pr["v"] = bf(pr["k"]), bf(pr["v"])
            kc[b, h], vc[b, h] = pr["k"], pr["v"]
            probs.append((b, h, pr))
    return dict(q=q.to(BF), kc=kc.to(BF), vc=vc.to(BF), pos0=c["pos0"], lens=c["lens"]), probs


# ---- decode_attn (bf16 and e4m3 caches): one new token per sample at position cur_len ----
def decode_splits(total, nsplit, e4m3):
    """The kernels' split ranges (attention.cu decode_attn_kernel / decode_attn_e4m3_kernel: chunk = ceil(total / nsplit),
    rounded up to a multiple of 4 keys on the e4m3 cache)."""
    chunk = (total + nsplit - 1) // nsplit
    if e4m3:
        chunk = (chunk + 3) // 4 * 4
    return [(min(s * chunk, total), min(s * chunk + chunk, total)) for s in range(nsplit)]


def mq_splits(total, nsplit):
    chunk = (total + nsplit - 1) // nsplit
    return [(min(s * chunk, total), min(s * chunk + chunk, total)) for s in range(nsplit)]


def nsplit_h100(B, H, Smax, ctas_per_sm):
    """model.cu decode_nsplit on 132 SMs with the kernels' resident CTAs per SM (6 / 4 / 3 for the bf16 / e4m3 / mq kernel,
    attention.cu *_ctas_per_sm). The GPU tests use b2_op_decode_attn_nsplit / _mq_nsplit, and when that value differs they
    repeat the sharpness check on the split edges it places."""
    n = min(max(ctas_per_sm * 132 // (B * H), 3), 16)
    return max(Smax // 64, 1) if n > Smax // 64 else n


def resolve_nsplit(c, lib=None):
    ns, B, H, Smax = c["nsplit"], len(c["lens"]), c["H"], c["Smax"]
    if ns != "auto":
        return ns
    e4m3 = c.get("kv") == "e4m3"
    if lib is None:
        return nsplit_h100(B, H, Smax, 4 if e4m3 else 6)
    from llava import _b2
    return int(lib.b2_op_decode_attn_nsplit(B, H, Smax, _b2.KV_E4M3 if e4m3 else _b2.KV_BF16))


def rope_rows_cpu(qkv, lens, H):
    """(q, k) roped at HF's rounding points, [B, H, 128] bf16 (stands in for the device RoPE on a CPU-only machine)."""
    v3 = qkv.view(qkv.shape[0], 3, H, 128)
    pos = torch.as_tensor(lens, dtype=torch.long)
    return KV.rope_bf16(v3[:, 0], pos), KV.rope_bf16(v3[:, 1], pos)


def build_decode(c, seed, nsplit):
    """qkv [B, 3*H*128] bf16 (pre-RoPE), the bf16 cache [B, H, Smax, 128] before the call (row cur_len holds poison: the
    kernel must attend the new token, not the stale row), and per (b, h) what the problem needs besides the roped rows."""
    lens, H, Smax, D = c["lens"], c["H"], c["Smax"], 128
    B = len(lens)
    e4m3 = c.get("kv") == "e4m3"
    g = torch.Generator().manual_seed(seed)
    scale = D ** -0.5
    qkv = torch.randn(B, 3, H, D, generator=g, dtype=F64)
    qkv[:, 0] = bf(qkv[:, 0])
    kc = torch.randn(B, H, Smax, D, generator=g, dtype=F64)
    vc = torch.randn(B, H, Smax, D, generator=g, dtype=F64)
    q_roped, _ = rope_rows_cpu(qkv.reshape(B, -1).to(BF), lens, H)
    plans = []
    for b in range(B):
        pos = lens[b]
        splits = decode_splits(pos + 1, nsplit, e4m3)
        for h in range(H):
            qr = q_roped[b, h].to(F64)
            edges = sorted({e - 1 for s, e in splits if e > s} - {pos})
            aims = [(pos - 1, 0, T_NEEDLE - 1.5)] + [(j, 0, T_NEEDLE - (i % 3)) for i, j in enumerate(edges)]
            if c["regime"] == "sink" and pos > 0:
                aims.append((0, 0, T_NEEDLE - 1))
            poison = [(0, j) for j in range(pos, min(pos + 3, Smax))]
            aims += [(j, 0, T_NEEDLE + 2) for _, j in poison]
            pr = _finish(g, qr[None], kc[b, h].clone(), vc[b, h].clone(), torch.tensor([pos]), torch.tensor([True]),
                         scale, aims, poison, set(edges) | {0}, c["regime"], splits)
            kc[b, h], vc[b, h] = pr["k"], pr["v"]
            # the new token: its pre-RoPE k aimed at the pre-RoPE q (a rotation by the same angle keeps the score)
            if c["regime"] != "flat":
                qp = qkv[b, 0, h]
                qkv[b, 1, h] = T_NEEDLE * qp / (scale * (qp * qp).sum())
                qkv[b, 2, h] = (_needle_v(g, pos, D, 10 * NEEDLE_V) + OFFSET_V if c["regime"] == "offset" else _needle_v(g, pos, D))
            pr["needles"] = sorted(set(pr["needles"]) | {pos}) if c["regime"] != "flat" else []
            pr["poison"] = [(0, j) for _, j in poison if j > pos] if c["regime"] != "flat" else []
            plans.append((b, h, pr))
    return dict(qkv=qkv.reshape(B, -1).to(BF), kc=kc.to(BF), vc=vc.to(BF), lens=lens), plans


def decode_problems(inp, plans, q_roped, k_new, e4m3):
    """Completes the decode problems with the roped q / new k rows ([B, H, 128] bf16) the kernel attends with. On the e4m3
    cache every key is the dequantised stored row, the appended one included."""
    H = inp["kc"].shape[1]
    v3 = inp["qkv"].view(inp["qkv"].shape[0], 3, H, 128)
    out = []
    for b, h, pr in plans:
        pos = inp["lens"][b]
        k = inp["kc"][b, h].clone()
        v = inp["vc"][b, h].clone()
        k[pos], v[pos] = k_new[b, h], v3[b, 2, h]
        if e4m3:
            k, v = (KV.dequantize_kv(*KV.quantize_kv(x)) for x in (k, v))
        out.append((b, h, dict(pr, q=q_roped[b, h].to(F64)[None], k=k.to(F64), v=v.to(F64))))
    return out


# ---- decode_attn_mq (the prompt-lookup verify step): R query rows at cur_len .. cur_len + R - 1 ----
def build_mq(c, seed, nsplit):
    """qkv [B*R, 3*H*128] (q already roped, as rope_kv_write_at leaves it), caches [B, H, Smax, 128] holding the rows'
    own K / V at cur_len + j."""
    lens, H, Smax, R, D = c["lens"], c["H"], c["Smax"], c["R"], 128
    B = len(lens)
    g = torch.Generator().manual_seed(seed)
    scale = D ** -0.5
    qkv = torch.randn(B, R, 3, H, D, generator=g, dtype=F64)
    qkv[:, :, 0] = bf(qkv[:, :, 0])
    kc = torch.randn(B, H, Smax, D, generator=g, dtype=F64)
    vc = torch.randn(B, H, Smax, D, generator=g, dtype=F64)
    probs = []
    for b in range(B):
        n = lens[b]
        splits = mq_splits(n + R, nsplit)
        qpos = n + torch.arange(R)
        for h in range(H):
            aims, poison = _diag_aims(qpos, range(R))
            edges = sorted({e - 1 for s, e in splits if e > s} - set(qpos.tolist()))
            aims += [(j, R - 1, T_NEEDLE - 0.5 - 0.5 * (i % 2)) for i, j in enumerate(edges)]
            if c["regime"] == "sink" and n > 0:
                aims += [(0, r, T_NEEDLE - 1) for r in range(R)]
            poison += [(R - 1, j) for j in range(n + R + 1, min(n + R + 3, Smax))]
            aims += [(j, R - 1, T_NEEDLE + 2) for r, j in poison[-2:] if j > n + R]
            pr = _finish(g, qkv[b, :, 0, h], kc[b, h].clone(), vc[b, h].clone(), qpos, torch.ones(R, dtype=torch.bool),
                         scale, aims, poison, set(edges) | set(qpos.tolist()), c["regime"], splits)
            pr["k"], pr["v"] = bf(pr["k"]), bf(pr["v"])
            kc[b, h], vc[b, h] = pr["k"], pr["v"]
            probs.append((b, h, pr))
    return dict(qkv=qkv.reshape(B * R, -1).to(BF), kc=kc.to(BF), vc=vc.to(BF), lens=lens), probs


# ------------------------------------------------------------------------------------------------------ the case table
FLASH_CASES = []
for _D in (64, 128):
    for _causal in (0, 1):
        FLASH_CASES += [dict(B=2, H=2, S=S, D=_D, causal=_causal, lens=None, regime="needle")
                        for S in (1, 63, 64, 65, 127, 128, 129, 257, 577)]
        FLASH_CASES += [dict(B=3, H=2, S=257, D=_D, causal=_causal, lens=[257, 1, 129], regime="needle"),
                        dict(B=2, H=2, S=577, D=_D, causal=_causal, lens=[577, 385], regime="offset"),
                        dict(B=2, H=2, S=577, D=_D, causal=_causal, lens=None, regime="flat")]
FLASH_CASES.append(dict(B=5, H=16, S=577, D=64, causal=0, lens=None, regime="needle"))  # five ViT images

FLASH_KV_CASES = [dict(S=S, H=2, pos0=[p0, p0 // 2 + 1], lens=[S, max(1, S // 2)], Smax=p0 + S + 64, regime="needle")
                  for p0 in (0, 1, 127, 128, 1000) for S in (1, 64, 129)]
FLASH_KV_CASES.append(dict(S=129, H=2, pos0=[300, 7], lens=[129, 100], Smax=600, regime="offset"))

DEC_LENS = [0, 1, 7, 8, 31, 32, 33]
DECODE_CASES = []
for _kv in ("bf16", "e4m3"):
    DECODE_CASES += [dict(kv=_kv, H=2, lens=DEC_LENS + [4095], Smax=4096, nsplit=ns, regime="needle") for ns in (1, "auto", 48)]
    DECODE_CASES += [dict(kv=_kv, H=2, lens=DEC_LENS, Smax=64, nsplit=40, regime="needle"),      # most splits empty
                     dict(kv=_kv, H=4, lens=[703, 1023, 64], Smax=1024, nsplit="auto", regime="sink"),
                     dict(kv=_kv, H=4, lens=[703, 1023, 64], Smax=1024, nsplit=7, regime="offset"),
                     dict(kv=_kv, H=4, lens=[703, 1023, 64], Smax=1024, nsplit=7, regime="flat")]

MQ_CASES = [dict(R=R, H=2, lens=[700, 130], Smax=1024, nsplit=ns, regime="needle") for R in (1, 2, 5, 16) for ns in (1, "auto", 9)]
MQ_CASES += [dict(R=R, H=2, lens=[1024 - R], Smax=1024, nsplit="auto", regime="needle") for R in (1, 5, 16)]  # cur_len + R = Smax
MQ_CASES += [dict(R=5, H=2, lens=[700, 64], Smax=1024, nsplit=5, regime="sink"),
             dict(R=16, H=2, lens=[700, 64], Smax=1024, nsplit=5, regime="offset"),
             dict(R=16, H=2, lens=[700, 64], Smax=1024, nsplit=5, regime="flat")]


def _cid(c):
    return "-".join(f"{k}{v}" for k, v in c.items()).replace(" ", "").replace("[", "").replace("]", "").replace(",", ".")


ALL_CASES = ([("flash", c) for c in FLASH_CASES] + [("flash_kv", c) for c in FLASH_KV_CASES] +
             [("decode", c) for c in DECODE_CASES] + [("mq", c) for c in MQ_CASES])


def cpu_problems(kind, c, seed=0):
    if kind == "flash":
        return build_flash(c, seed)[1]
    if kind == "flash_kv":
        return build_flash_kv(c, seed)[1]
    if kind == "mq":
        return build_mq(c, seed, nsplit_h100(1, c["H"], c["Smax"], 3) if c["nsplit"] == "auto" else c["nsplit"])[1]
    inp, plans = build_decode(c, seed, resolve_nsplit(c))
    q, k = rope_rows_cpu(inp["qkv"], inp["lens"], c["H"])
    return decode_problems(inp, plans, q, k, c["kv"] == "e4m3")


# ------------------------------------------------------------------------------------------------------ CPU self-check
@pytest.mark.parametrize("kind,case", ALL_CASES, ids=[f"{k}-{_cid(c)}" for k, c in ALL_CASES])
def test_mutated_references_violate_the_bound(kind, case):
    """Every plausible wrong answer falls outside the bound, on every (sample, head) of every case with needles. (The flat
    cases are the unit-randn control, run on the GPU only.)"""
    if case["regime"] == "flat":
        pytest.skip("flat control")
    assert_sharp(cpu_problems(kind, case))


def assert_sharp(probs, heads=2):
    """Every mutation of every problem (heads 0 .. heads-1) that changes the answer at all falls outside the bound."""
    escaped, total = [], 0
    for b, h, pr in probs:
        if h >= heads:
            continue
        ref, p = attend(pr)
        assert worst_ratio(pr, ref, ref, p) == 0.0
        for name, mut in mutations(pr).items():
            got, _ = attend(pr, **mut)
            if float((got - ref)[pr["rows"]].abs().max()) <= 1e-9 * (1.0 + float(ref.abs().max())):
                continue  # the mutation changes nothing this problem computes (e.g. a shift past every checked row)
            total += 1
            if worst_ratio(pr, got, ref, p) <= 1.0:
                escaped.append(f"b{b} h{h}: {name}")
    assert total > 0 and not escaped, escaped[:10]


# ------------------------------------------------------------------------------------------------------ GPU: op level
@pytest.fixture(scope="module")
def lib():
    from llava import _b2

    _b2.init(0)
    return _b2.load_library()


def _P(t):
    from llava import _b2
    return _b2.ptr(t)


def _S():
    from llava import _b2
    return _b2.stream_ptr()


def _check_problems(kind, case, probs, out_of):
    worst = 0.0
    for b, h, pr in probs:
        ref, p = attend(pr)
        got = out_of(b, h).to(F64).cpu()
        assert torch.isfinite(got[pr["rows"]]).all(), (kind, b, h)
        r = worst_ratio(pr, got, ref, p)
        worst = max(worst, r)
        assert r <= 1.0, f"{kind} b{b} h{h}: err/bound {r:.3f} (> 1 at kappa = {KAPPA})"
    print(f"\n[attention-numerics] {kind} {_cid(case)}: worst err/bound {worst:.4f}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", FLASH_CASES, ids=[_cid(c) + "-wgmma" for c in FLASH_CASES])
def test_flash_attn(lib, case):
    from llava import _b2

    inp, probs = build_flash(case, seed=1)
    B, S, H, D = case["B"], case["S"], case["H"], case["D"]
    q, k, v = (inp[n].to(DEV) for n in ("q", "k", "v"))
    lens = None if inp["lens"] is None else torch.tensor(inp["lens"], device=DEV, dtype=torch.int32)
    o = torch.full_like(q, float("nan"))
    _b2.check(lib.b2_op_flash_attn(_P(q), _P(k), _P(v), _P(o), _P(lens), B, S, H, D, case["causal"], D ** -0.5, _S()))
    o = o.cpu()
    _check_problems("flash_wgmma", case, probs, lambda b, h: o[b, :, h])


@pytest.mark.gpu
@pytest.mark.parametrize("case", FLASH_KV_CASES, ids=[_cid(c) for c in FLASH_KV_CASES])
def test_flash_attn_kv(lib, case):
    from llava import _b2

    inp, probs = build_flash_kv(case, seed=2)
    B, S, H = len(case["pos0"]), case["S"], case["H"]
    q, kc, vc = (inp[n].to(DEV) for n in ("q", "kc", "vc"))
    pos0 = torch.tensor(inp["pos0"], device=DEV, dtype=torch.int32)
    lens = torch.tensor(inp["lens"], device=DEV, dtype=torch.int32)
    o = torch.full_like(q, float("nan"))
    _b2.check(lib.b2_op_flash_attn_kv(_P(q), _P(kc), _P(vc), _P(o), _P(pos0), _P(lens), B, S, H, case["Smax"], 128 ** -0.5, _S()))
    o = o.cpu()
    _check_problems("flash_kv", case, probs, lambda b, h: o[b, :, h])


def _device_rope(lib, qkv, lens, H, Smax):
    """q / k of each row roped at its cur_len by b2_op_rope_kv_write_at (the RoPE code the decode kernels run): [B, H, 128]."""
    B = qkv.shape[0]
    x = qkv.clone().to(DEV)
    kd = torch.zeros(B, H, Smax, 128, device=DEV, dtype=BF)
    vd = torch.zeros_like(kd)
    pos = torch.tensor(lens, device=DEV, dtype=torch.int32)
    from llava import _b2
    _b2.check(lib.b2_op_rope_kv_write_at(_P(x), _P(kd), _P(vd), _P(pos), B, 1, H, 128, Smax, 10000.0, _S()))
    k = torch.stack([kd[b, :, lens[b]] for b in range(B)]).cpu()
    return x.view(B, 3, H, 128)[:, 0].cpu(), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", DECODE_CASES, ids=[_cid(c) for c in DECODE_CASES])
def test_decode_attn(lib, case):
    from llava import _b2

    e4m3 = case["kv"] == "e4m3"
    nsplit = resolve_nsplit(case, lib)
    inp, plans = build_decode(case, seed=3, nsplit=nsplit)
    lens, H, Smax = inp["lens"], case["H"], case["Smax"]
    B = len(lens)
    q_roped, k_new = _device_rope(lib, inp["qkv"], lens, H, Smax)
    probs = decode_problems(inp, plans, q_roped, k_new, e4m3)
    if case["regime"] != "flat" and nsplit != resolve_nsplit(case):
        assert_sharp(probs)  # the CPU self-check placed split-edge needles for another split factor
    qkv = inp["qkv"].to(DEV)
    cur = torch.tensor(lens, device=DEV, dtype=torch.int32)
    scratch = torch.zeros(lib.b2_op_decode_attn_scratch_bytes(B, H, nsplit), device=DEV, dtype=torch.uint8)
    out = torch.full((B, H * 128), float("nan"), device=DEV, dtype=BF)
    if e4m3:
        cache = KV.empty_cache(B, H, Smax)
        KV.store_rows(cache, inp["kc"], inp["vc"])
        c0 = {n: t.to(DEV) for n, t in cache.items()}
    else:
        c0 = dict(kc=inp["kc"].to(DEV), vc=inp["vc"].to(DEV))
    for _ in range(2):  # the second launch runs on the split counters the first one left behind
        dev = {n: t.clone() for n, t in c0.items()}
        if e4m3:
            _b2.check(lib.b2_op_decode_attn_e4m3(_P(qkv), _P(dev["k8"]), _P(dev["v8"]), _P(dev["ks"]), _P(dev["vs"]), _P(cur),
                                                 _P(out), _P(scratch), B, H, Smax, nsplit, 10000.0, 128 ** -0.5, _S()))
        else:
            _b2.check(lib.b2_op_decode_attn(_P(qkv), _P(dev["kc"]), _P(dev["vc"]), _P(cur), _P(out), _P(scratch), B, H, Smax,
                                            nsplit, 10000.0, 128 ** -0.5, _S()))
    assert int(scratch[: B * H * 4].view(torch.int32).abs().sum()) == 0, "split counters must be left at zero"
    o = out.view(B, H, 128).cpu()
    _check_problems("decode_" + case["kv"], case, probs, lambda b, h: o[b, h][None])
    # the cache append: exactly row cur_len written, with the roped k and the v of qkv (quantised on the e4m3 cache)
    v_new = inp["qkv"].view(B, 3, H, 128)[:, 2]
    for b in range(B):
        n = lens[b]
        if e4m3:
            for name, sname, x in (("k8", "ks", k_new[b]), ("v8", "vs", v_new[b])):
                q8, s = KV.quantize_kv(x)
                got8, gots = dev[name].cpu(), dev[sname].cpu()
                assert torch.equal(got8[b, :, n].view(torch.uint8), q8.view(torch.uint8)) and torch.equal(gots[b, :, n], s)
                assert torch.equal(got8[b, :, :n].view(torch.uint8), c0[name][b, :, :n].cpu().view(torch.uint8))
                assert torch.equal(got8[b, :, n + 1:].view(torch.uint8), c0[name][b, :, n + 1:].cpu().view(torch.uint8))
        else:
            kc, vc = dev["kc"].cpu(), dev["vc"].cpu()
            assert torch.equal(kc[b, :, n], k_new[b]) and torch.equal(vc[b, :, n], v_new[b])
            assert torch.equal(kc[b, :, :n], inp["kc"][b, :, :n]) and torch.equal(kc[b, :, n + 1:], inp["kc"][b, :, n + 1:])
            assert torch.equal(vc[b, :, :n], inp["vc"][b, :, :n]) and torch.equal(vc[b, :, n + 1:], inp["vc"][b, :, n + 1:])


@pytest.mark.gpu
@pytest.mark.parametrize("case", MQ_CASES, ids=[_cid(c) for c in MQ_CASES])
def test_decode_attn_mq(lib, case):
    from llava import _b2

    if case["nsplit"] == "auto":
        nsplit = int(lib.b2_op_decode_attn_mq_nsplit(case["H"], case["Smax"]))
    else:
        nsplit = case["nsplit"]
    inp, probs = build_mq(case, seed=4, nsplit=nsplit)
    if case["regime"] != "flat" and case["nsplit"] == "auto" and nsplit != nsplit_h100(1, case["H"], case["Smax"], 3):
        assert_sharp(probs)  # the CPU self-check placed split-edge needles for another split factor
    lens, H, Smax, R = inp["lens"], case["H"], case["Smax"], case["R"]
    B = len(lens)
    qkv, kc, vc = (inp[n].to(DEV) for n in ("qkv", "kc", "vc"))
    scratch = torch.zeros(lib.b2_op_decode_attn_mq_scratch_bytes(B, H, nsplit), device=DEV, dtype=torch.uint8)
    cur = torch.tensor(lens, device=DEV, dtype=torch.int32)
    out = torch.full((B * R, H * 128), float("nan"), device=DEV, dtype=BF)
    for _ in range(2):
        _b2.check(lib.b2_op_decode_attn_mq(_P(qkv), _P(kc), _P(vc), _P(cur), _P(out), _P(scratch), B, R, H, Smax, nsplit,
                                           128 ** -0.5, _S()))
    o = out.view(B, R, H, 128).cpu()
    _check_problems("mq", case, probs, lambda b, h: o[b, :, h])

# ------------------------------------------------------------------------------------------------------ GPU: RoPE rows
# Relative difference of the kernels' RoPE angle pos * exp2f(-(2i/D) log2f(theta)) from HF's pos * (1 / theta^(2i/D)): the
# fp32 inv_freq differ by up to 4.9e-7 (numpy fp32 restatement of the device formula), CUDA's exp2f / log2f add up to 2 ulp
# each (2 * 2^-23), and each side's fp32 product rounds by 2^-24: 8.5e-7 in all, under 2^-20.
ANGLE_REL = 2.0 ** -20
ROPE_POS = sorted(set(range(0, 4096, 31)) | {1, 63, 64, 127, 128, 4094, 4095})


def _rope_rows(lib, e4m3):
    """The K rows of one 4096-token prefill chunk (b2_op_rope_kv_write_at at pos0 = 0, then on the e4m3 cache
    b2_op_kv_quantize_e4m3 of those rows) and the rows one decode step appends at each position of ROPE_POS (one sample per
    position, fed the same pre-RoPE k)."""
    from llava import _b2

    H, Smax, n = 2, 4096, len(ROPE_POS)
    g = torch.Generator().manual_seed(9)
    k_pre = torch.randn(Smax, H * 128, generator=g).to(BF)
    qkv = torch.randn(Smax, 3, H * 128, generator=g).to(BF)
    qkv[:, 1] = k_pre
    qkv = qkv.to(DEV)
    kc = torch.zeros(1, H, Smax, 128, device=DEV, dtype=BF)
    vc = torch.zeros_like(kc)
    zero = torch.zeros(1, device=DEV, dtype=torch.int32)
    _b2.check(lib.b2_op_rope_kv_write_at(_P(qkv), _P(kc), _P(vc), _P(zero), 1, Smax, H, 128, Smax, 10000.0, _S()))
    dq = qkv[torch.tensor(ROPE_POS, device=DEV)].reshape(n, -1).clone()
    cur = torch.tensor(ROPE_POS, device=DEV, dtype=torch.int32)
    scratch = torch.zeros(lib.b2_op_decode_attn_scratch_bytes(n, H, 4), device=DEV, dtype=torch.uint8)
    out = torch.empty(n, H * 128, device=DEV, dtype=BF)
    if not e4m3:
        kd, vd = torch.zeros(n, H, Smax, 128, device=DEV, dtype=BF), torch.zeros(n, H, Smax, 128, device=DEV, dtype=BF)
        _b2.check(lib.b2_op_decode_attn(_P(dq), _P(kd), _P(vd), _P(cur), _P(out), _P(scratch), n, H, Smax, 4, 10000.0,
                                        128 ** -0.5, _S()))
        return [(kc[0, :, p], kd[i, :, p]) for i, p in enumerate(ROPE_POS)]
    k8 = torch.zeros(1, H, Smax, 128, device=DEV, dtype=torch.uint8)
    v8, ks, vs = torch.zeros_like(k8), torch.zeros(1, H, Smax, device=DEV), torch.zeros(1, H, Smax, device=DEV)
    _b2.check(lib.b2_op_kv_quantize_e4m3(_P(kc), _P(vc), _P(k8), _P(v8), _P(ks), _P(vs), None, 1, Smax, H, Smax, _S()))
    k8d = torch.zeros(n, H, Smax, 128, device=DEV, dtype=torch.uint8)
    v8d, ksd, vsd = torch.zeros_like(k8d), torch.zeros(n, H, Smax, device=DEV), torch.zeros(n, H, Smax, device=DEV)
    _b2.check(lib.b2_op_decode_attn_e4m3(_P(dq), _P(k8d), _P(v8d), _P(ksd), _P(vsd), _P(cur), _P(out), _P(scratch), n, H, Smax,
                                         4, 10000.0, 128 ** -0.5, _S()))
    return [((k8[0, :, p], ks[0, :, p]), (k8d[i, :, p], ksd[i, :, p])) for i, p in enumerate(ROPE_POS)]


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["bf16", "e4m3"])
def test_prefill_and_decode_write_bit_identical_k_rows(lib, kv):
    """The K row a prefill stores for position p is the row a decode step appends at p: a cache filled by either path
    is attended the same way."""
    for p, (pre, dec) in zip(ROPE_POS, _rope_rows(lib, kv == "e4m3")):
        if kv == "e4m3":
            assert torch.equal(pre[0], dec[0]) and torch.equal(pre[1], dec[1]), p
        else:
            assert torch.equal(pre, dec), p


@pytest.mark.gpu
def test_rope_cos_sin_within_one_bf16_ulp_of_hf(lib):
    """The kernels' (cos, sin) (inv_freq = exp2(-(2i/D) log2(theta)) in fp32) against HF's 1 / theta^(2i/D): read back by
    roping k = [1]*64 + [0]*64, whose rotated halves are exactly the bf16 cos and sin. At most one bf16 ulp apart anywhere."""
    from llava import _b2

    Smax = 4096
    qkv = torch.zeros(Smax, 3, 128, device=DEV, dtype=BF)
    qkv[:, 1, :64] = 1.0
    kc = torch.zeros(1, 1, Smax, 128, device=DEV, dtype=BF)
    vc = torch.zeros_like(kc)
    zero = torch.zeros(1, device=DEV, dtype=torch.int32)
    _b2.check(lib.b2_op_rope_kv_write_at(_P(qkv), _P(kc), _P(vc), _P(zero), 1, Smax, 1, 128, Smax, 10000.0, _S()))
    got = kc[0, 0].cpu()                                                    # [Smax, 128]: cos | sin
    cos, sin = O._rope_cos_sin(torch.arange(Smax)[None], 128, 10000.0, BF)
    want = torch.cat([cos[0, :, :64], sin[0, :, :64]], -1)
    got, want = got.double(), want.double()
    diff = (got - want).abs()
    mag = torch.maximum(got.abs(), want.abs()).clamp(min=2.0 ** -126)
    ulp = 2.0 ** (torch.floor(torch.log2(mag)) - 7)
    # the angles pos * inv_freq_i of the two formulas differ by up to ang * ANGLE_REL; near a zero crossing of cos / sin that is
    # more than a bf16 ulp of the tiny value, so it is allowed on top of the one ulp of rounding (per frequency: at the low
    # frequencies the angle, and with it the allowance, stays small)
    inv = 1.0 / 10000.0 ** (torch.arange(0, 128, 2, dtype=torch.float64) / 128)
    ang = torch.arange(Smax, dtype=torch.float64)[:, None] * inv[None, :]
    allowed = ulp + torch.cat([ang, ang], -1) * ANGLE_REL
    print(f"\n[attention-numerics] RoPE cos/sin differ from HF's in {100 * float((diff > 0).double().mean()):.2f} % of "
          f"(position, frequency) entries ({int((diff[:64] > 0).sum())} below position 64); more than one bf16 ulp apart: "
          f"{int((diff > ulp).sum())}, largest difference {float(diff.max()):.2e}")
    assert bool((diff <= allowed).all()), float((diff / allowed).max())


# ------------------------------------------------------------------------------------------------------ model level
# The megakernel's attention phase (decode_mega.cu mk_attention) has no op entry, so it and every other decode path run on
# weights that put each head's mass on the query's own key: k_proj += DIAG_GAIN * q_proj. RoPE cancels at relative distance 0,
# so a row's score with its own key is DIAG_GAIN * |q|^2 / sqrt(d) ~ 7 (unit-gain linears: |q|^2 ~ d), while its scores with
# the other keys stay ~N(0, 1.2). In a decode step the own key is the new token, the one key every decode kernel handles apart
# from the cache. The prefill is long enough that the megakernel's split of the key range over G CTAs (G = SMs / heads = 66
# on the tiny config) puts several keys in each CTA, and the new token sits at the end of the last one.
DIAG_GAIN, PROMPT_LEN, N_STEPS, MAX_SEQ = 0.6, 230, 3, 320
# e4m3 cache against the restated quantised step (max, mean of the logit std). The engine's cache holds the e4m3 codes of its
# bf16 prefill's K / V, the restatement those of the fp32 oracle's: an element whose two values round to neighbouring codes is
# off by one e4m3 step (2^-4 relative). The restatement filled from the bf16 oracle's prefill is itself 0.097 / 0.018 away
# (H100 run of this file), above test_kv_fp8_gpu's KERNEL_TOL (0.08 / 0.015), whose cache is the same on both sides.
E4M3_TOL = (0.15, 0.03)
CFG = O.CONFIGS["tiny"]


def sharp_weights(cfg, seed=0):
    w = O.make_weights(cfg, seed=seed)
    for i in range(cfg["layers"]):
        p = f"model.layers.{i}.self_attn."
        w[p + "k_proj.weight"] = (w[p + "k_proj.weight"] + DIAG_GAIN * w[p + "q_proj.weight"]).to(BF).float()
    return w


def _prompt(cfg, w, B, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, cfg["vocab"], (B, PROMPT_LEN), generator=g)
    return w["model.embed_tokens.weight"][ids], torch.randint(0, cfg["vocab"], (B, N_STEPS + 1), generator=g)


def _forward(w, x, drop_own_last=False):
    """fp32 decoder over x [1, S, h] (O.llama_forward's math): (last row's logits, attention weights per layer). With
    drop_own_last the last row does not attend its own key in any layer: a decode step that leaves out the new token."""
    F = torch.nn.functional
    H, S = CFG["heads"], x.shape[1]
    d = CFG["hidden"] // H
    cos, sin = O._rope_cos_sin(torch.arange(S)[None], d, CFG["rope_theta"], torch.float32)
    mask = torch.triu(torch.full((S, S), -math.inf), 1)
    if drop_own_last:
        mask[S - 1, S - 1] = -math.inf
    ps = []
    for i in range(CFG["layers"]):
        W = lambda k: w[f"model.layers.{i}.{k}"]
        y = O._rmsnorm(x, W("input_layernorm.weight"), CFG["rms_eps"])
        q, k, v = (F.linear(y, W(f"self_attn.{n}_proj.weight")).view(1, S, H, d).transpose(1, 2) for n in ("q", "k", "v"))
        q, k = q * cos[:, None] + O._rotate_half(q) * sin[:, None], k * cos[:, None] + O._rotate_half(k) * sin[:, None]
        p = torch.softmax((q @ k.transpose(2, 3)) * d ** -0.5 + mask, -1)
        ps.append(p[0])
        x = x + F.linear((p @ v).transpose(1, 2).reshape(1, S, -1), W("self_attn.o_proj.weight"))
        y = O._rmsnorm(x, W("post_attention_layernorm.weight"), CFG["rms_eps"])
        x = x + F.linear(F.silu(F.linear(y, W("mlp.gate_proj.weight"))) * F.linear(y, W("mlp.up_proj.weight")),
                         W("mlp.down_proj.weight"))
    x = O._rmsnorm(x, w["model.norm.weight"], CFG["rms_eps"])
    return F.linear(x[:, -1], w["lm_head.weight"]), ps


def test_sharp_weights_put_the_mass_on_the_own_key():
    """From the oracle's own q / k: in every (layer, head) the median over query rows of the weight on the row's own key
    exceeds 0.5, and a decode step that leaves the new token out moves the logits far outside the GPU tests' tolerances
    (mean error 1 % of std against the oracle, 0.6 % against a prefill recompute)."""
    from helpers import rel_err

    w = sharp_weights(CFG)
    emb, toks = _prompt(CFG, w, 1, seed=8)
    x = torch.cat([emb, w["model.embed_tokens.weight"][toks[:, :1]]], 1)
    logits, ps = _forward(w, x)
    for i, p in enumerate(ps):
        own = p.diagonal(dim1=-2, dim2=-1).median(-1).values      # [H]
        assert bool((own > 0.5).all()), (i, own.tolist())
    dropped, _ = _forward(w, x, drop_own_last=True)
    mx, mn = rel_err(dropped, logits)
    assert mn > 0.03 and mx > 0.15, (mx, mn)


# id: (kv dtype, B, R): R = rows of one b2_decode_rows call instead of N_STEPS decode steps
MODEL_PATHS = {"mega-b1": ("bf16", 1, 0), "gemv-b4": ("bf16", 4, 0), "streamk-b12": ("bf16", 12, 0), "e4m3-b1": ("e4m3", 1, 0),
               "decode-rows-r4": ("bf16", 1, 4)}


@pytest.fixture(scope="module")
def sharp_engine():
    from helpers import make_engine

    w = sharp_weights(CFG)
    eng = make_engine(CFG, w, max_batch=12, max_seq=MAX_SEQ, max_images=1)
    yield w, eng
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", list(MODEL_PATHS))
def test_sharp_attention_decode_paths(sharp_engine, path):
    """Step logits against the fp32 oracle with the model tests' rule (5 % / 1 % of the logit std, and a mean error within
    2x the oracle's own bf16 noise + 2e-3) and against a prefill that recomputes the same positions with the path tests'
    3 % / 0.6 %; on the e4m3 cache against the restated quantised step (oracle/kv_fp8_oracle.py) with E4M3_TOL and the same
    mean rule."""
    from llava import _b2
    from test_model_gpu import _check

    kv_dtype, B, R = MODEL_PATHS[path]
    if path == "gemv-b4" and os.environ.get("B2_DECODE_MEGA") != "0":
        pytest.skip("runs in a process without the megakernel: test_sharp_attention_gemv_graph")
    w, eng = sharp_engine
    emb, toks = _prompt(CFG, w, B, seed=7 + B)
    kv = eng.new_kv(B, MAX_SEQ, dtype=kv_dtype)
    eng.prefill(kv, emb.to(DEV), None, _b2.LOGITS_LAST)
    E = w["model.embed_tokens.weight"]
    if R:
        got = eng.decode_rows(kv, toks[0, :R]).cpu()[None]               # [1, R, V]
        ref, _ = O.llama_forward(w, torch.cat([emb, E[toks[:, :R]]], 1), CFG)
        bref, _ = O.llama_forward(w, torch.cat([emb, E[toks[:, :R]]], 1), CFG, dtype=BF)
        _check(f"{path} rows", got, ref[:, -R:], bf16_ref=bref[:, -R:])
        kv.close()
        return
    if kv_dtype == "e4m3":  # the restated quantised cache, filled by the fp32 and by the bf16 oracle prefill
        _, caches = KV.prefill_cache(w, emb, CFG, MAX_SEQ)
        bcaches = []
        for k, v in O.llama_forward(w, emb, CFG, dtype=BF, last_only=True)[1]:
            c = KV.empty_cache(B, CFG["heads"], MAX_SEQ)
            KV.store_rows(c, k, v)
            bcaches.append(c)
    _, ref_kv = O.llama_forward(w, emb, CFG, last_only=True)
    _, bref_kv = O.llama_forward(w, emb, CFG, dtype=BF, last_only=True)
    for t in range(N_STEPS):
        tok = toks[:, t]
        before = _b2.launch_count()
        got = eng.decode_step(kv, tok.to(torch.int32).to(DEV)).cpu()
        torch.cuda.synchronize()
        launches = _b2.launch_count() - before
        if path == "mega-b1" and t > 0:  # (the cache's first step also uploads the sampling state)
            assert launches <= 2, launches  # the megakernel (plus at most the sampling tail), not the 13-launch GEMV step
        ref, ref_kv = O.llama_forward(w, E[tok][:, None], CFG, kv=ref_kv, last_only=True)
        bref, bref_kv = O.llama_forward(w, E[tok][:, None], CFG, kv=bref_kv, dtype=BF, last_only=True)
        if kv_dtype == "e4m3":
            want = KV.decode_step(w, tok, CFG, caches, [PROMPT_LEN + t] * B)
            bwant = KV.decode_step(w, tok, CFG, bcaches, [PROMPT_LEN + t] * B, dtype=BF)
            _check(f"{path} step {t} vs quantised oracle", got, want, bf16_ref=bwant, tol_max=E4M3_TOL[0], tol_mean=E4M3_TOL[1])
        else:
            _check(f"{path} step {t}", got, ref[:, -1], bf16_ref=bref[:, -1])
        if kv_dtype == "bf16":
            # against a prefill that recomputes every position from scratch (not on the e4m3 cache: its decode attends the
            # stored quantised rows, its prefill the unquantised K / V)
            rc = eng.new_kv(B, MAX_SEQ)
            recompute = eng.prefill(rc, torch.cat([emb, E[toks[:, :t + 1]]], 1).to(DEV), None, _b2.LOGITS_LAST).cpu()
            rc.close()
            _check(f"{path} step {t} vs prefill recompute", got, recompute, tol_max=0.03, tol_mean=0.006)
    kv.close()


@pytest.mark.gpu
def test_sharp_attention_gemv_graph(repo_root):
    """The bf16 GEMV graph at batch 4, in a process started with B2_DECODE_MEGA=0 (read once per process)."""
    env = dict(os.environ, B2_DECODE_MEGA="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "test_sharp_attention_decode_paths and gemv-b4"],
                       cwd=repo_root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "1 passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
