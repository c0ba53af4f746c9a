"""Every attention kernel (csrc/attention.cu) checked element by element against fp64: o, lse, dQ, dK and dV of every
forward / backward entry point, at the shapes, masks and inputs where a mask edge, a tile walk or a head mapping goes
wrong, against the bounds of numerics.attention_reference / attention_bwd_reference.

The five entry-point pairs launch 17 kernel instantiations between them; KERNELS maps each pair to the ones it launches
(checked against the launchers in attention.cu), and a test asserts that the cases below reach all 17.  Every batch row
holds a different layout and every case has at least 3 query heads where the entry point allows, so a batch or head
indexing error shows.  Inputs come in three families: randn; peaky (q and k x3, so |s| reaches about 30 and exp2
underflows for part of each row); late max (a ramp along the key axis puts each row's largest scores in its last visible
tile, so every tile rescales the running sums).

Cross-checks that need no tolerance: grouped-query attention with kv_heads == heads is multi-head attention bitwise
(o, lse and dqkv: the grouped dK / dV loop is a hand-kept copy of the multi-head one), and grouped-query attention equals
multi-head attention on K / V repeated per group bitwise in o, lse and dQ, at head dims 64 and 128.
"""
import os
import re

import pytest
import torch

import numerics as nm
from b200ddp.ops.functional import window_bounds
from test_gpu_causal_attention import LAYOUTS

pytestmark = pytest.mark.gpu

KERNELS = {                                                     # entry point -> the instantiations it launches
    "attention": ("attn_fwd_kernel<kKeyPadding>", "attn_bwd_dot_kernel", "attn_bwd_dkdv_kernel<kKeyPadding>",
                  "attn_bwd_dq_kernel<kKeyPadding>"),
    "packed_attention": ("attn_fwd_kernel<kSegment>", "attn_bwd_dot_kernel", "attn_bwd_dkdv_kernel<kSegment>",
                         "attn_bwd_dq_kernel<kSegment>"),
    "causal_attention": ("attn_fwd_kernel<kCausal>", "attn_bwd_dot_kernel", "attn_bwd_dkdv_kernel<kCausal>",
                         "attn_bwd_dq_kernel<kCausal>"),
    "causal_gqa_attention": ("attn_fwd_kernel<kCausal, true>", "attn_bwd_dot_kernel", "attn_bwd_dkdv_kernel<kCausal, true>",
                             "attn_bwd_dq_kernel<kCausal, true>"),
    "causal_attention_d128": ("attn_fwd_d128_kernel", "attn_bwd_dot_d128_kernel", "attn_bwd_dkdv_d128_kernel",
                              "attn_bwd_dq_d128_kernel"),
}
GROUP = {"attention": "key_padding", "packed_attention": "packed", "causal_attention": "causal",
         "causal_gqa_attention": "gqa", "causal_attention_d128": "d128"}
SCALE = {64: 0.125, 128: float(torch.tensor(0.08838834764831845, dtype=torch.float32))}   # kScale, kScale128 (fp32)
FAMILIES = ("randn", "peaky", "late_max")


def _rows(S):
    """Every row of every LAYOUTS layout at S, one layout row per batch row."""
    return [row for name in sorted(LAYOUTS) for row in LAYOUTS[name](S)]


def _lens(S):
    return [0, 1, 2, 63, 64, 65, 127, 128, 129, S - 1, S]


# (entry point, S, heads, kv_heads, mask, window): mask "lens" (seq_lens), "layouts" (bounds of _rows(S)) or "one_doc"
CASES = ([("attention", S, 3, 3, "lens", None) for S in (128, 256, 640)]
         + [("packed_attention", S, 3, 3, "layouts", None) for S in (256, 640)]
         + [("packed_attention", 640, 3, 3, "layouts", w) for w in (1, 63, 64, 127, 128, 200, 639)]
         + [("causal_attention", S, 3, 3, "layouts", None) for S in (256, 640, 2048)]
         + [("causal_gqa_attention", 640, H, Hkv, "layouts", None) for H, Hkv in ((4, 1), (4, 2), (6, 3), (9, 3), (4, 4))]
         + [("causal_attention_d128", 640, H, Hkv, "layouts", None) for H, Hkv in ((2, 2), (4, 2), (6, 1), (16, 8))])
LONG_CASE = ("packed_attention", 8192, 2, 2, "one_doc", 64)   # ModernBERT's local attention at its full length


def _case_id(case):
    entry, S, H, Hkv, mask, w = case
    return f"{entry}-S{S}-H{H}" + (f"-kv{Hkv}" if Hkv != H else "") + (f"-w{w}" if w is not None else "")


def test_cases_reach_every_kernel_instantiation():
    src = open(os.path.join(os.path.dirname(__file__), os.pardir, "b200ddp", "csrc", "attention.cu")).read()
    # the launchers: attention_fwd<kMode[, true]>("<entry>_fwd", ...) and the d128 pair's own kernels
    for args, entry in re.findall(r"attention_fwd<([^>]+)>\(\"(\w+)_fwd\"", src):
        assert KERNELS[entry][0] == f"attn_fwd_kernel<{args}>", entry
    for args, entry in re.findall(r"attention_bwd<([^>]+)>\(\"(\w+)_bwd\"", src):
        assert KERNELS[entry][2:] == (f"attn_bwd_dkdv_kernel<{args}>", f"attn_bwd_dq_kernel<{args}>"), entry
    d128 = re.search(r"void launch_causal_attention_d128_bwd.*?\n}\n", src, re.S).group(0)
    assert set(re.findall(r"(attn_\w+_kernel)<<<", d128)) == set(KERNELS["causal_attention_d128"][1:])
    every = {k for ks in KERNELS.values() for k in ks}
    assert len(every) == 17
    assert {k for case in CASES + [LONG_CASE] for k in KERNELS[case[0]]} == every


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


def _mask(kind, S, window=None):
    """The mask on the GPU: seq_lens int32 [B] ("lens") or bounds int32 [B, S, 2], windowed when `window` is given."""
    if kind == "lens":
        return torch.tensor(_lens(S), dtype=torch.int32, device="cuda")
    rows = _rows(S) if kind == "layouts" else [[S]]
    b = torch.zeros(len(rows), S, 2, dtype=torch.int32)
    for r, docs in enumerate(rows):
        at = 0
        for n in docs:
            b[r, at:at + n, 0], b[r, at:at + n, 1] = at, at + n
            at += n
    b = b.cuda()
    return b if window is None else window_bounds(b, window)


def _qkv(B, S, H, Hkv, d, family, seed):
    """qkv bf16 [B*S, (H + 2 Hkv) d] and dout bf16 [B*S, H d]."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, S, H + 2 * Hkv, d, device="cuda", generator=g)
    if family == "peaky":
        x[:, :, :H + Hkv] *= 3
    elif family == "late_max":
        x[:, :, :H, 0] = 4.0
        x[:, :, H:H + Hkv, 0] = (torch.arange(S, device="cuda") - S / 2)[None, :, None] / 16
    dout = torch.randn(B * S, H * d, device="cuda", generator=g)
    return x.reshape(B * S, -1).to(torch.bfloat16), dout.to(torch.bfloat16)


def _heads(t, B, S, d):
    """[B*S, n*d] -> [B, n, S, d]"""
    return t.reshape(B, S, -1, d).transpose(1, 2)


def _split(t, B, S, H, Hkv, d):
    x = _heads(t, B, S, d)
    return x[:, :H], x[:, H:H + Hkv], x[:, H + Hkv:]


def _run(C, entry, qkv, mask, dout, H, Hkv):
    """(o, lse, dqkv) of one forward and backward entry-point pair."""
    extra = (Hkv,) if entry in ("causal_gqa_attention", "causal_attention_d128") else ()
    o, lse = getattr(C, entry + "_fwd")(qkv, mask, H, *extra)
    dqkv = getattr(C, entry + "_bwd")(dout, qkv, o, lse, mask, H, *extra)
    return o, lse, dqkv


def _check_case(C, case, family, seed):
    entry, S, H, Hkv, kind, window = case
    d = 128 if entry == "causal_attention_d128" else 64
    mask = _mask(kind, S, window)
    B = mask.shape[0]
    qkv, dout = _qkv(B, S, H, Hkv, d, family, seed)
    o, lse, dqkv = _run(C, entry, qkv, mask, dout, H, Hkv)
    q, k, v = _split(qkv, B, S, H, Hkv, d)
    vis = nm.attention_visible(mask, S, causal=entry.startswith("causal"))
    where = f"{_case_id(case)} {family}"
    group = f"attn {GROUP[entry]}"
    fwd = nm.attention_reference(q, k, v, vis, SCALE[d])
    nm.check_attention(where, {"o": _heads(o, B, S, d), "lse": lse}, fwd, group)
    del fwd                                                     # the fp64 references are the largest tensors here
    bwd = nm.attention_bwd_reference(q, k, v, _heads(o, B, S, d), lse, _heads(dout, B, S, d), vis, SCALE[d])
    dq, dk, dv = _split(dqkv, B, S, H, Hkv, d)
    nm.check_attention(where, {"dq": dq, "dk": dk, "dv": dv}, bwd, group)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_attention_matches_fp64_elementwise(C, case, family):
    _check_case(C, case, family, seed=3 * CASES.index(case) + FAMILIES.index(family))


@pytest.mark.parametrize("family", ["randn", "late_max"])
def test_modernbert_length_window_matches_fp64_on_every_row(C, family):
    _check_case(C, LONG_CASE, family, seed=5)


@pytest.mark.parametrize("S", [640, 2048])
def test_gqa_with_kv_heads_equal_to_heads_is_multi_head_bitwise(C, S):
    H = 3
    mask = _mask("layouts", S)
    qkv, dout = _qkv(mask.shape[0], S, H, H, 64, "randn", seed=S)
    mha = _run(C, "causal_attention", qkv, mask, dout, H, H)
    gqa = _run(C, "causal_gqa_attention", qkv, mask, dout, H, H)
    for name, a, b in zip(("o", "lse", "dqkv"), mha, gqa):
        assert torch.equal(a, b), f"{name}: grouped-query attention with kv_heads == heads differs from multi-head attention"


@pytest.mark.parametrize("entry,d,H,Hkv", [("causal_gqa_attention", 64, 4, 2), ("causal_gqa_attention", 64, 9, 3),
                                           ("causal_attention_d128", 128, 4, 2), ("causal_attention_d128", 128, 6, 1)])
def test_gqa_is_multi_head_attention_on_repeated_kv_bitwise(C, entry, d, H, Hkv):
    S = 640
    mask = _mask("layouts", S)
    B = mask.shape[0]
    qkv, dout = _qkv(B, S, H, Hkv, d, "randn", seed=H * Hkv)
    q, k, v = _split(qkv, B, S, H, Hkv, d)
    g = H // Hkv
    rep = torch.cat([q, k.repeat_interleave(g, 1), v.repeat_interleave(g, 1)], 1)
    qkv_mha = rep.transpose(1, 2).reshape(B * S, 3 * H * d).contiguous()
    o, lse, dqkv = _run(C, entry, qkv, mask, dout, H, Hkv)
    mha = "causal_attention" if d == 64 else entry
    o_m, lse_m, dqkv_m = _run(C, mha, qkv_mha, mask, dout, H, H)
    assert torch.equal(o, o_m), "o"
    assert torch.equal(lse, lse_m), "lse"
    assert torch.equal(dqkv[:, :H * d], dqkv_m[:, :H * d]), "dq"
