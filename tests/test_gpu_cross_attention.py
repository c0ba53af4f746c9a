"""The cross-attention kernels (csrc/cross_attention.cu) checked element by element against fp64: o, lse, dQ, dK and dV
against the bounds of numerics.attention_reference / attention_bwd_reference, at query and key lengths that differ.
Those references take one length for both sides, so each case runs them on S = max(Sq, Sk): queries past Sq and keys
past Sk are padding that nothing sees (lse -inf, zero o and dO), which adds exact zeros to every sum and leaves the
real rows' references and bounds as they are.

Every batch row holds a different layout of (source, target) document pairs: one pair whose lengths walk 0, 1, 63, 64,
65, 127, 128, 129, S - 1 and S on each side, packed rows of several pairs, a target document whose source is empty, a
source that no target sees, and an all-padding row.  Inputs come in the three families of test_gpu_attention_elementwise
(randn, peaky, late max).  Also: the backward is bitwise repeatable, ``ops.cross_attention`` matches its own CPU
reference and a dense-mask SDPA, and malformed inputs raise ``ValueError``.
"""
import os
import random
import re

import pytest
import torch
import torch.nn.functional as F

import numerics as nm
from b200ddp.ops import cross_attention, cross_bounds, document_bounds
from b200ddp.ops.functional import cross_attention_reference

pytestmark = pytest.mark.gpu

SHAPES = [(128, 128), (256, 640), (640, 256), (1024, 1024)]   # (Sq, Sk)
FAMILIES = ("randn", "peaky", "late_max")
H = 3
D = 64
SCALE = 0.125
KERNELS = {"cross_fwd_kernel", "attn_bwd_dot_kernel", "cross_dkdv_kernel", "cross_dq_kernel"}


def _lens(S):
    return [0, 1, 63, 64, 65, 127, 128, 129, S - 1, S]


def _layouts(Sq, Sk):
    """Rows of (source length, target length) pairs, laid out back to back on each side."""
    rows = [[(s, t)] for s, t in zip(_lens(Sk), reversed(_lens(Sq)))]   # every length on each side, mismatched partners
    rows += [[(s, s)] for s in (1, 65, min(Sq, Sk))]
    rng = random.Random(Sq * 7 + Sk)
    for _ in range(2):                                          # packed rows of random pairs
        pairs, a, b = [], 0, 0
        while True:
            s, t = rng.randint(0, 150), rng.randint(1, 150)
            if a + s > Sk or b + t > Sq:
                break
            pairs.append((s, t))
            a, b = a + s, b + t
        rows.append(pairs)
    rows.append([(40, 30), (0, 50), (1, 1), (64, 0), (20, 20)])   # an empty source, a source without a target
    rows.append([])                                             # all padding
    return rows


def _bounds(rows, Sq, Sk):
    """(q_bounds [B, Sq, 2], kv_bounds [B, Sk, 2]) int32 on the GPU: target k of a row sees source k."""
    qb = torch.zeros(len(rows), Sq, 2, dtype=torch.int32)
    kb = torch.zeros(len(rows), Sk, 2, dtype=torch.int32)
    for r, pairs in enumerate(rows):
        a = b = 0
        for s, t in pairs:
            qb[r, b:b + t, 0], qb[r, b:b + t, 1] = a, a + s
            kb[r, a:a + s, 0], kb[r, a:a + s, 1] = b, b + t
            a, b = a + s, b + t
    return qb.cuda(), kb.cuda()


def _inputs(B, Sq, Sk, family, seed):
    """q bf16 [B*Sq, H*64], kv bf16 [B*Sk, 2*H*64], dout bf16 [B*Sq, H*64]."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, Sq, H, D, device="cuda", generator=g)
    kv = torch.randn(B, Sk, 2 * H, D, device="cuda", generator=g)
    if family == "peaky":
        q *= 3
        kv[:, :, :H] *= 3
    elif family == "late_max":
        q[..., 0] = 4.0
        kv[:, :, :H, 0] = (torch.arange(Sk, device="cuda") - Sk / 2)[None, :, None] / 16
    dout = torch.randn(B * Sq, H * D, device="cuda", generator=g)
    return (q.reshape(B * Sq, -1).to(torch.bfloat16), kv.reshape(B * Sk, -1).to(torch.bfloat16), dout.to(torch.bfloat16))


def _heads(t, B, S):
    """[B*S, n*64] -> [B, n, S, 64]"""
    return t.reshape(B, S, -1, D).transpose(1, 2)


def _visible(qb, Sk):
    """[B, Sq, Sk] bool: query i sees key j iff q_bounds' start <= j < end (start clamped to [0, Sk], end to [start, Sk],
    as the kernels' row_bounds does)."""
    b = qb.long()
    start = b[..., 0].clamp(0, Sk)
    end = torch.maximum(b[..., 1], start).clamp(max=Sk)
    j = torch.arange(Sk, device=qb.device)
    return (j >= start[..., None]) & (j < end[..., None])


def _square(t, S, fill=0.0):
    """[B, n, L, ...] padded along dim 2 to S rows of `fill`"""
    pad = t.new_full((t.shape[0], t.shape[1], S - t.shape[2], *t.shape[3:]), fill)
    return torch.cat([t, pad], 2)


def _check(where, Sq, Sk, qh, k, v, o, lse, dout, dq, dk, dv, vis):
    """numerics' fp64 references and bounds on the problem padded to S = max(Sq, Sk), checked on the real rows."""
    S = max(Sq, Sk)
    B = qh.shape[0]
    sq = torch.zeros(B, S, S, dtype=torch.bool, device=vis.device)
    sq[:, :Sq, :Sk] = vis
    Q, K, V, O, dO = (_square(t, S) for t in (qh, k, v, o, dout))
    fwd = nm.attention_reference(Q, K, V, sq, SCALE)
    fwd = {key: tuple(t[:, :, :Sq] for t in pair) for key, pair in fwd.items()}
    nm.check_attention(where, {"o": o, "lse": lse}, fwd, "attn cross")
    del fwd
    bwd = nm.attention_bwd_reference(Q, K, V, O, _square(lse, S, -float("inf")), dO, sq, SCALE)
    bwd = {key: tuple(t[:, :, :(Sq if key == "dq" else Sk)] for t in pair) for key, pair in bwd.items()}
    nm.check_attention(where, {"dq": dq, "dk": dk, "dv": dv}, bwd, "attn cross")


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


def test_cases_reach_every_kernel():
    src = open(os.path.join(os.path.dirname(__file__), os.pardir, "b200ddp", "csrc", "cross_attention.cu")).read()
    defined = set(re.findall(r"__global__ void __launch_bounds__\(\w+, 1\)\s+(\w+)\(", src))
    assert defined == KERNELS - {"attn_bwd_dot_kernel"}        # the dot kernel is attention_common.cuh's
    assert set(re.findall(r"(\w+_kernel)<<<", src)) == KERNELS
    # every pair of lengths, each launcher reaches its kernels' early exits (all-padding rows) and their full paths
    for Sq, Sk in SHAPES:
        rows = _layouts(Sq, Sk)
        assert [] in rows and any(t > 0 and s == 0 for r in rows for s, t in r) and any(s > 0 and t == 0 for r in rows for s, t in r)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("Sq,Sk", SHAPES)
def test_cross_attention_matches_fp64_elementwise(C, Sq, Sk, family):
    rows = _layouts(Sq, Sk)
    B = len(rows)
    qb, kb = _bounds(rows, Sq, Sk)
    q, kv, dout = _inputs(B, Sq, Sk, family, seed=Sq + 3 * Sk + FAMILIES.index(family))
    o, lse = C.cross.cross_attention_fwd(q, kv, qb, H)
    dq, dkv = C.cross.cross_attention_bwd(dout, q, kv, o, lse, qb, kb, H)
    kvh, dkvh = _heads(kv, B, Sk), _heads(dkv, B, Sk)
    _check(f"cross Sq{Sq} Sk{Sk} {family}", Sq, Sk, _heads(q, B, Sq), kvh[:, :H], kvh[:, H:], _heads(o, B, Sq), lse,
           _heads(dout, B, Sq), _heads(dq, B, Sq), dkvh[:, :H], dkvh[:, H:], _visible(qb, Sk))


def test_backward_is_bitwise_repeatable(C):
    Sq, Sk = 256, 640
    rows = _layouts(Sq, Sk)
    qb, kb = _bounds(rows, Sq, Sk)
    q, kv, dout = _inputs(len(rows), Sq, Sk, "randn", seed=11)
    o, lse = C.cross.cross_attention_fwd(q, kv, qb, H)
    first = C.cross.cross_attention_bwd(dout, q, kv, o, lse, qb, kb, H)
    second = C.cross.cross_attention_bwd(dout, q, kv, o, lse, qb, kb, H)
    assert torch.equal(first[0], second[0]) and torch.equal(first[1], second[1])


def test_op_matches_reference_and_dense_sdpa():
    """ops.cross_attention on bounds from cross_bounds of packed rows: the fp32 reference on the CPU and SDPA with the
    dense mask, forward and both gradients."""
    torch.manual_seed(0)
    Sq, Sk, B = 256, 384, 3
    src = torch.full((B, Sk), 0)
    tgt = torch.full((B, Sq), 0)
    src[0, :300], tgt[0, :200] = 5, 5                           # one pair
    src[1, :100], src[1, 100:250], tgt[1, :90], tgt[1, 90:256] = 5, 5, 5, 5
    src[1, 100], tgt[1, 90] = 9, 9                              # two pairs
    src[2, :7], tgt[2, :3] = 5, 5
    enc, _ = document_bounds(src, 9, 0)
    dec, _ = document_bounds(tgt, 9, 0)
    qb, kb = cross_bounds(enc.cuda(), dec.cuda())
    q = torch.randn(B, Sq, H * D, device="cuda").bfloat16().requires_grad_()
    kv = torch.randn(B, Sk, 2 * H * D, device="cuda").bfloat16().requires_grad_()
    g = torch.randn(B, Sq, H * D, device="cuda").bfloat16()
    out = cross_attention(q, kv, qb, kb, H)
    dq, dkv = torch.autograd.grad(out, (q, kv), g)
    qf, kvf = q.detach().float().cpu().requires_grad_(), kv.detach().float().cpu().requires_grad_()
    ref = cross_attention(qf, kvf, qb.cpu(), kb.cpu(), H)
    rdq, rdkv = torch.autograd.grad(ref, (qf, kvf), g.float().cpu())
    keep = _visible(qb, Sk)[:, None]
    qs = q.detach().float().view(B, Sq, H, D).transpose(1, 2)
    k, v = (t.view(B, Sk, H, D).transpose(1, 2) for t in kv.detach().float().split(H * D, -1))
    sdpa = F.scaled_dot_product_attention(qs, k, v, attn_mask=keep).nan_to_num(0.0) * keep.any(-1, keepdim=True)
    sdpa = sdpa.transpose(1, 2).reshape(B, Sq, H * D)
    for name, got, want in (("o", out.detach(), ref.detach()), ("o vs sdpa", out.detach(), sdpa.cpu()), ("dq", dq, rdq), ("dkv", dkv, rdkv)):
        err = nm.rel_err(got.float().cpu(), want)
        assert err < 1e-2, f"{name}: relative error {err:.3g}"
    assert torch.equal(cross_attention_reference(qf.detach(), kvf.detach(), qb.cpu(), H), ref.detach())


@pytest.mark.parametrize("change,match", [
    (lambda q, kv, qb, kb: (q.float(), kv, qb, kb), "bf16"),
    (lambda q, kv, qb, kb: (q[:, :100], kv, qb[:, :100], kb), "multiples of 128"),
    (lambda q, kv, qb, kb: (q, kv[..., :-64], qb, kb), r"kv \[B, Sk, 2 \* hidden\]"),
    (lambda q, kv, qb, kb: (q.transpose(0, 1).contiguous().transpose(0, 1), kv, qb, kb), "contiguous"),
    (lambda q, kv, qb, kb: (q, kv, kb, kb), "q_bounds"),
    (lambda q, kv, qb, kb: (q, kv, qb, kb.float()), "kv_bounds"),
])
def test_op_rejects_what_the_kernels_cannot_run(change, match):
    q = torch.zeros(2, 128, H * D, device="cuda", dtype=torch.bfloat16)
    kv = torch.zeros(2, 256, 2 * H * D, device="cuda", dtype=torch.bfloat16)
    qb = torch.zeros(2, 128, 2, device="cuda", dtype=torch.int32)
    kb = torch.zeros(2, 256, 2, device="cuda", dtype=torch.int32)
    with pytest.raises(ValueError, match=match):
        cross_attention(*change(q, kv, qb, kb), H)
