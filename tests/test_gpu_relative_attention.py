"""T5's relative position bias inside the attention kernels (csrc/attention.cu, kBias) checked element by element
against fp64: o, lse, dQ, dK, dV and dtable of both bias instantiations (segment and causal), on every layout of
test_gpu_causal_attention.LAYOUTS (documents longer than S are cut at S) at S in {128, 384, 640, 1024}, so tiles wholly
beyond +-128 occur on both sides, with 3 heads and the three input families of the other attention tests.

The references follow numerics.attention_reference / attention_bwd_reference with the scores unscaled and the fp32 bias
added (one more rounding of each score); dtable sums the fp32 dS of each clamped distance, bounded by the per-term dS
error plus the kernels' longest fp32 summation chain.  Also here: bitwise repeatable backwards (dqkv, dtable and
d weight), T5's unscaled cross-attention as cross_attention(8 q, ...), and the bias-free ReLU linear on the wgmma GEMM.
"""
import math
import os
import re

import pytest
import torch

import numerics as nm
from test_gpu_causal_attention import LAYOUTS

pytestmark = pytest.mark.gpu

H, D = 3, 64
FAMILIES = ("randn", "peaky", "late_max")
SEQS = (128, 384, 640, 1024)
KERNELS = {"attn_fwd_kernel<kMode, false, true>", "attn_bwd_dot_kernel", "attn_bwd_dkdv_kernel<kMode, false, true>",
           "attn_bwd_dq_kernel<kMode, false, true>", "rel_bias_finish_kernel"}


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


def _rows(S):
    """Every row of every LAYOUTS layout at S, its documents cut where they pass S."""
    out = []
    for name in sorted(LAYOUTS):
        for docs in LAYOUTS[name](S):
            row, at = [], 0
            for n in docs:
                n = min(n, S - at)
                if n > 0:
                    row.append(n)
                    at += n
            out.append(row)
    return out


def _bounds(rows, S):
    b = torch.zeros(len(rows), S, 2, dtype=torch.int32)
    for r, docs in enumerate(rows):
        at = 0
        for n in docs:
            b[r, at:at + n, 0], b[r, at:at + n, 1] = at, at + n
            at += n
    return b.cuda()


def _inputs(B, S, family, seed):
    """qkv bf16 [B*S, 3*H*64], dout bf16 [B*S, H*64], table fp32 [H, 257] (a different value in every column)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, S, 3 * H, D, device="cuda", generator=g)
    if family == "peaky":
        x[:, :, :2 * H] *= 3
    elif family == "late_max":
        x[:, :, :H, 0] = 4.0
        x[:, :, H:2 * H, 0] = (torch.arange(S, device="cuda") - S / 2)[None, :, None] / 16
    dout = torch.randn(B * S, H * D, device="cuda", generator=g)
    table = 2 * torch.randn(H, 257, device="cuda", generator=g)
    return x.reshape(B * S, -1).to(torch.bfloat16), dout.to(torch.bfloat16), table


def _heads(t, B, S):
    return t.reshape(B, S, -1, D).transpose(1, 2)


def _cols(M, S):
    """[H, S, S] (query, key) -> [H, 257]: the sums over each clamped distance key - query."""
    out = torch.zeros(M.shape[0], 257, dtype=torch.float64, device=M.device)
    for d in range(-min(127, S - 1), min(127, S - 1) + 1):
        out[:, d + 128] = torch.diagonal(M, offset=d, dim1=-2, dim2=-1).sum(-1)
    out[:, 0] = torch.tril(M, -128).sum((-1, -2))
    out[:, 256] = torch.triu(M, 128).sum((-1, -2))
    return out


def _reference(q, k, v, table, o, lse, dout, vis):
    """fp64 forward and backward of one batch row (q, k, v, o, dout [H, S, d]; lse [H, S]; vis [S, S]) with the bias, and
    the bounds of the kernels' arithmetic, as numerics' attention references derive them at scale 1.  Returns
    {"o", "lse", "dq", "dk", "dv"}: (ref, acc) and "dtable": (ref, bound)."""
    c, e, U, BU = nm.C_ACC, nm.EXP_ULPS, nm.U, nm.BF16_U
    S = q.shape[1]
    Q, K, V, O, dO = (t.double() for t in (q, k, v, o, dout))
    pos = torch.arange(S, device=q.device)
    s = Q @ K.transpose(-1, -2) + table.double()[:, (pos[None, :] - pos[:, None]).clamp(-128, 128) + 128]
    A = c * D * U * (Q.abs() @ K.abs().transpose(-1, -2))
    visf = vis[None]
    n = vis.sum(-1).double()[None]
    tiles = vis.reshape(S, S // nm.KEY_TILE, nm.KEY_TILE).any(-1).sum(-1).double()[None]
    l = torch.logsumexp(s.masked_fill(~visf, -math.inf), -1)
    live = torch.isfinite(l)
    P = torch.where(visf, torch.exp(s - torch.where(live, l, 0.0)[..., None]), 0.0)
    smax = torch.where(visf, s.abs(), 0.0).amax(-1, keepdim=True)
    rho = A + U * (e + 4 + 2 * (s.abs() + smax)) + (e + 3) * U * tiles[..., None]
    Prho = P * rho
    sum_prho = Prho.sum(-1)
    oc = P @ V
    Va = V.abs()
    out = {"o": (oc, (BU * P + Prho) @ Va + (c * U * (n + 1))[..., None] * (P @ Va) + oc.abs() * (sum_prho + (n + 2) * U)[..., None]),
           "lse": (l, torch.where(live, sum_prho + (n + 2) * U + 2 * U * (torch.where(live, l, 0.0).abs() + 1), 0.0))}
    # backward at the kernel's own o and lse
    L = lse.double()
    live = torch.isfinite(L)
    Lz = torch.where(live, L, 0.0)[..., None]
    visb = visf & live[..., None]
    P = torch.where(visb, torch.exp(s - Lz), 0.0)
    dP = dO @ V.transpose(-1, -2)
    err_dP = c * D * U * (dO.abs() @ Va.transpose(-1, -2))
    Dr = (dO * O).sum(-1, keepdim=True)
    err_D = D * U * (dO * O).abs().sum(-1, keepdim=True)
    dS = P * (dP - Dr)
    rho = A + U * (e + 4 + 2 * (s.abs() + Lz.abs()))
    err_pre = P * rho * (dP - Dr).abs() + P * (err_dP + err_D) + 2 * U * dS.abs()
    err_dS = err_pre + BU * (dS.abs() + err_pre)
    err_P = P * (rho + BU * (1 + rho))
    dSa, Ka = dS.abs(), K.abs()
    n = visb.sum(-1).double()
    m = visb.sum(-2).double()[..., None]
    out["dq"] = (dS @ K, err_dS @ Ka + (U * c * (n + 1))[..., None] * (dSa @ Ka))
    out["dk"] = (dS.transpose(-1, -2) @ Q, err_dS.transpose(-1, -2) @ Q.abs() + U * c * (m + 1) * (dSa.transpose(-1, -2) @ Q.abs()))
    out["dv"] = (P.transpose(-1, -2) @ dO, err_P.transpose(-1, -2) @ dO.abs() + c * U * (m + 1) * (P.transpose(-1, -2) @ dO.abs()))
    out["dtable"] = (_cols(dS, S), _cols(err_pre, S), _cols(dSa, S))
    return out


def _check(C, S, causal, family, seed):
    rows = _rows(S)
    B = len(rows)
    bounds = _bounds(rows, S)
    qkv, dout, table = _inputs(B, S, family, seed)
    o, lse = C.t5.relative_attention_fwd(qkv, bounds, table, H, causal)
    dqkv, dtable = C.t5.relative_attention_bwd(dout, qkv, o, lse, bounds, table, H, causal)
    vis = nm.attention_visible(bounds, S, causal=causal)
    x, dx, oh, dOh = _heads(qkv, B, S), _heads(dqkv, B, S), _heads(o, B, S), _heads(dout, B, S)
    where = f"relative {'causal' if causal else 'segment'} S{S} {family}"
    # the longest fp32 chain a dtable term goes through: slot fold, the owner's 64 slots or the far sums of every tile's
    # 18 slots, the warp and CTA reduction, the finish over (b, query tile)
    depth = 2 + 64 + 18 * (S // 64) + 13 + B * (S // 128)
    dt_ref = torch.zeros(H, 257, dtype=torch.float64, device="cuda")
    dt_err = torch.zeros_like(dt_ref)
    dt_mag = torch.zeros_like(dt_ref)
    for b in range(B):
        ref = _reference(x[b, :H], x[b, H:2 * H], x[b, 2 * H:], table, oh[b], lse[b], dOh[b], vis[b])
        got = {"o": oh[b:b + 1], "lse": lse[b:b + 1], "dq": dx[b:b + 1, :H], "dk": dx[b:b + 1, H:2 * H], "dv": dx[b:b + 1, 2 * H:]}
        nm.check_attention(f"{where} row {b}", got, {k: tuple(t[None] for t in ref[k]) for k in got})
        r, err, mag = ref["dtable"]
        dt_ref += r
        dt_err += err
        dt_mag += mag
    nm.check(f"{where}: dtable [h, c]", dtable, dt_ref, dt_err + depth * nm.U * dt_mag + nm.FLOOR)


def test_cases_reach_every_new_kernel():
    src = open(os.path.join(os.path.dirname(__file__), os.pardir, "b200ddp", "csrc", "attention.cu")).read()
    body = re.search(r"void relative_bwd\(.*?\n}\n", src, re.S).group(0) + re.search(r"void relative_fwd\(.*?\n}\n", src, re.S).group(0)
    assert set(re.findall(r"(\w+_kernel(?:<[^>]*>)?)<<<", body)) == KERNELS
    assert re.search(r'relative_fwd<kCausal>\("relative_attention_fwd"', src) and re.search(r'relative_fwd<kSegment>\("relative_attention_fwd"', src)
    assert re.search(r'relative_bwd<kCausal>\("relative_attention_bwd"', src) and re.search(r'relative_bwd<kSegment>\("relative_attention_bwd"', src)
    for S in SEQS:                                              # tiles beyond +-128 on both sides, empty and padding rows
        rows = _rows(S)
        assert [] in rows and any(sum(r) < S for r in rows) and (S < 384 or any(max(r, default=0) >= 384 for r in rows))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("S", SEQS)
@pytest.mark.parametrize("causal", [False, True], ids=["segment", "causal"])
def test_relative_attention_matches_fp64_elementwise(C, causal, S, family):
    _check(C, S, causal, family, seed=S + FAMILIES.index(family) + 7 * causal)


@pytest.mark.parametrize("causal", [False, True], ids=["segment", "causal"])
def test_backward_is_bitwise_repeatable(causal):
    from b200ddp.ops import relative_attention, relative_position_table
    S = 640
    rows = _rows(S)
    bounds = _bounds(rows, S)
    qkv, dout, _ = _inputs(len(rows), S, "randn", seed=3)
    w = (torch.randn(32, H, device="cuda") * 2).to(torch.bfloat16)
    grads = []
    for _ in range(2):
        x = qkv.view(len(rows), S, -1).clone().requires_grad_(True)
        wt = w.clone().requires_grad_(True)
        table = relative_position_table(wt, bidirectional=not causal)
        table.retain_grad()
        relative_attention(x, bounds, table, H, causal).backward(dout.view(len(rows), S, -1))
        grads.append((x.grad, table.grad, wt.grad))
    for name, a, b in zip(("dqkv", "dtable", "d weight"), *grads):
        assert torch.equal(a, b), name


def test_table_fold_matches_fp64():
    from b200ddp.ops import relative_position_bucket, relative_position_table
    for bidirectional in (True, False):
        w = torch.randn(32, H, device="cuda", requires_grad=True)
        dt = torch.randn(H, 257, device="cuda")
        table = relative_position_table(w, bidirectional)
        idx = relative_position_bucket(torch.arange(-128, 129), bidirectional).cuda()
        assert torch.equal(table, w.detach()[idx].t())
        table.backward(dt)
        ref = torch.zeros(32, H, dtype=torch.float64, device="cuda").index_add_(0, idx, dt.double().t())
        count = torch.bincount(idx, minlength=32).double()[:, None]
        nm.check("d weight", w.grad, ref, count * nm.U * torch.zeros_like(ref).index_add_(0, idx, dt.double().abs().t()) + nm.FLOOR)


def test_op_matches_dense_reference():
    """relative_attention on CUDA (bf16) against its fp32 dense reference, through autograd: qkv and table gradients."""
    from b200ddp.ops import relative_attention, relative_attention_reference
    S = 384
    rows = _rows(S)
    B = len(rows)
    bounds = _bounds(rows, S)
    qkv, dout, table = _inputs(B, S, "randn", seed=9)
    x = (qkv.view(B, S, -1).float() / 4).to(torch.bfloat16)     # T5-like score magnitudes
    for causal in (False, True):
        a, ta = x.clone().requires_grad_(True), table.clone().requires_grad_(True)
        out = relative_attention(a, bounds, ta, H, causal)
        out.backward(dout.view(B, S, -1))
        r, tr = x.float().clone().requires_grad_(True), table.clone().requires_grad_(True)
        ref = relative_attention_reference(r, bounds, tr, H, causal)
        ref.backward(dout.view(B, S, -1).float())
        for name, got, want in (("o", out.detach().float(), ref.detach()), ("dqkv", a.grad.float(), r.grad), ("dtable", ta.grad, tr.grad)):
            rel = float((got - want).norm() / want.norm())
            assert rel < 2e-2, (causal, name, rel)


def test_cross_attention_times_eight_is_unscaled_attention(C):
    """T5's cross-attention has no 1/sqrt(d) scale: cross_attention(8 q, ...) is it, since 8 q is exact in bf16 and the
    kernel's 1/8 undoes the 8 exactly.  The kernels on 8 q (and 8 dq', autograd's factor) meet numerics' fp64 bounds of
    the unscaled attention of q."""
    import test_gpu_cross_attention as tc
    Sq, Sk = 256, 640
    rows = tc._layouts(Sq, Sk)
    B = len(rows)
    qb, kb = tc._bounds(rows, Sq, Sk)
    q, kv, dout = tc._inputs(B, Sq, Sk, "randn", seed=21)
    q = (q.float() / 8).to(torch.bfloat16)                      # unscaled scores of T5's magnitude
    q8 = q * 8
    assert torch.equal(q8.float(), q.float() * 8)
    o, lse = C.cross.cross_attention_fwd(q8, kv, qb, tc.H)
    dq8, dkv = C.cross.cross_attention_bwd(dout, q8, kv, o, lse, qb, kb, tc.H)
    dq = dq8 * 8
    assert torch.equal(dq.float(), dq8.float() * 8)
    S = max(Sq, Sk)
    sq = torch.zeros(B, S, S, dtype=torch.bool, device="cuda")
    sq[:, :Sq, :Sk] = tc._visible(qb, Sk)
    kvh = tc._heads(kv, B, Sk)
    Q, K, V, O, dO = (tc._square(t, S) for t in (tc._heads(q, B, Sq), kvh[:, :tc.H], kvh[:, tc.H:], tc._heads(o, B, Sq), tc._heads(dout, B, Sq)))
    fwd = nm.attention_reference(Q, K, V, sq, 1.0)
    nm.check_attention("cross x8 fwd", {"o": tc._heads(o, B, Sq), "lse": lse}, {k: tuple(t[:, :, :Sq] for t in p) for k, p in fwd.items()})
    bwd = nm.attention_bwd_reference(Q, K, V, O, tc._square(lse, S, -float("inf")), dO, sq, 1.0)
    dkvh = tc._heads(dkv, B, Sk)
    got = {"dq": tc._heads(dq, B, Sq), "dk": dkvh[:, :tc.H], "dv": dkvh[:, tc.H:]}
    nm.check_attention("cross x8 bwd", got, {k: tuple(t[:, :, :(Sq if k == "dq" else Sk)] for t in p) for k, p in bwd.items()})


def test_bias_free_relu_linear_runs_on_the_wgmma_gemm():
    from torch.profiler import ProfilerActivity, profile

    from b200ddp.ops import linear
    torch.manual_seed(0)
    x = torch.randn(512, 768, device="cuda").to(torch.bfloat16)
    w = (torch.randn(3072, 768, device="cuda") * 0.05).to(torch.bfloat16)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        y = linear(x, w, None, "relu")
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("gemm_bf16_kernel" in n for n in names), names                  # the wgmma GEMM, ReLU in its epilogue
    assert not any(t in n.lower() for n in names for t in ("relu", "clamp", "xmma", "nvjet", "cutlass", "cublas")), names
    ref, acc = nm.gemm_reference(x, w, torch.zeros(3072, device="cuda", dtype=torch.bfloat16), 2)
    nm.check("bias-free relu linear", y, ref, nm.bound(ref, acc, y.dtype))
