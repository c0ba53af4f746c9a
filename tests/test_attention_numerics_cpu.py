"""The attention bounds of numerics.py, on the CPU, against an emulation of the kernels' arithmetic (csrc/attention.cu):
the emulation stays well inside every bound on causal, packed, windowed and key-padding masks at head dims 64 and 128,
and each fault a mask edge, a tile walk, a head mapping or a store could plausibly make fails, including single-row mask
faults that the older global-norm checks let through.

The emulation follows the kernels step by step in fp32: scores on key tiles of 128 with an online softmax (exp2 against
the running maximum, one rescale per tile, P rounded to bf16 for P V, the fp32 row sum of the unrounded p); dK / dV over
64-query tiles, the query heads of a group in turn into one accumulator; dQ over 64-key tiles; P' and dS rounded to bf16,
D from the bf16 o; the scale applied to dK and dQ when they are stored."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import numerics as nm
from b200ddp.ops.functional import window_bounds

LOG2E = float(np.float32(1.4426950408889634))
SCALE = {64: float(np.float32(0.125)), 128: float(np.float32(0.08838834764831845))}   # kScale, kScale128


def _scale_log2(d):
    return float(np.float32(SCALE[d]) * np.float32(LOG2E))


def emulate_fwd(q, k, v, vis, kv_head=None):
    """(o bf16 [B, H, S, d], lse fp32 [B, H, S]) as the forward kernels compute them; vis [B, S, S] or [B, H, S, S]."""
    B, H, S, d = q.shape
    kv_head = kv_head or [h // (H // k.shape[1]) for h in range(H)]
    Q, K, V = q.float(), k[:, kv_head].float(), v[:, kv_head].float()
    vis = vis if vis.dim() == 4 else vis[:, None]
    cl2 = _scale_log2(d)
    m = torch.full((B, H, S), -math.inf)
    l = torch.zeros(B, H, S)
    acc = torch.zeros(B, H, S, d)
    for t in range(0, S, 128):
        s = (Q @ K[:, :, t:t + 128].transpose(-1, -2)).masked_fill(~vis[..., t:t + 128], -math.inf)
        mx = torch.maximum(m, s.amax(-1))
        base = torch.where(mx == -math.inf, 0.0, mx)            # no visible key yet: exp2 gives 0 rather than NaN
        alpha = torch.exp2((m - base) * cl2)
        m = mx
        p = torch.exp2(s * cl2 - (base * cl2)[..., None])
        l = l * alpha + p.sum(-1)
        acc = acc * alpha[..., None] + p.bfloat16().float() @ V[:, :, t:t + 128]
    o = (acc * torch.where(l > 0, 1.0 / l, 0.0)[..., None]).bfloat16()
    return o, torch.where(l > 0, m * SCALE[d] + torch.log(l), -math.inf)


def emulate_bwd(q, k, v, o, lse, dout, vis, drop_stage=None, first_head_only=False, d_head=None):
    """(dq, dk, dv) bf16 as the backward kernels compute them.  Faults: drop_stage = (b, key tile of 128) skips that
    tile's last 64-query ring stage in dK / dV; first_head_only sums only each group's first query head into dK / dV;
    d_head[h] is the head whose D query head h uses."""
    B, H, S, d = q.shape
    Hkv = k.shape[1]
    g = H // Hkv
    vis = (vis if vis.dim() == 4 else vis[:, None]).expand(B, H, S, S)
    cl2 = _scale_log2(d)
    Q, K, V, dO = q.float(), k.float(), v.float(), dout.float()
    D = (dO * o.float()).sum(-1)
    if d_head is not None:
        D = D[:, d_head]
    L2 = torch.where(torch.isneginf(lse), math.inf, lse * LOG2E)   # a query that saw no key gets P = 0
    dk, dv = torch.zeros(B, Hkv, S, d), torch.zeros(B, Hkv, S, d)
    last = None
    if drop_stage is not None:                                  # the key tile's last query tile with a visible entry
        b, kt = drop_stage
        seen = vis[b, :, :, kt * 128:(kt + 1) * 128].any(-1).any(0).nonzero()
        last = int(seen.max()) // 64
    for j in range(1 if first_head_only else g):
        h = [hk * g + j for hk in range(Hkv)]
        for t in range(0, S, 64):
            st = K @ Q[:, h, t:t + 64].transpose(-1, -2)        # [B, Hkv, keys, 64 queries]
            dpt = V @ dO[:, h, t:t + 64].transpose(-1, -2)
            keep = vis[:, h, t:t + 64].transpose(-1, -2).clone()
            if last is not None and t // 64 == last and j == g - 1:
                keep[b, :, kt * 128:(kt + 1) * 128] = False
            p = torch.where(keep, torch.exp2(st * cl2 - L2[:, h, None, t:t + 64]), 0.0)
            ds = p * (dpt - D[:, h, None, t:t + 64])
            dv = dv + p.bfloat16().float() @ dO[:, h, t:t + 64]
            dk = dk + ds.bfloat16().float() @ Q[:, h, t:t + 64]
    Kh, Vh = K.repeat_interleave(g, 1), V.repeat_interleave(g, 1)
    dq = torch.zeros(B, H, S, d)
    for t in range(0, S, 64):
        s = Q @ Kh[:, :, t:t + 64].transpose(-1, -2)
        dp = dO @ Vh[:, :, t:t + 64].transpose(-1, -2)
        p = torch.where(vis[..., t:t + 64], torch.exp2(s * cl2 - L2[..., None]), 0.0)
        ds = p * (dp - D[..., None])
        dq = dq + ds.bfloat16().float() @ Kh[:, :, t:t + 64]
    return (dq * SCALE[d]).bfloat16(), (dk * SCALE[d]).bfloat16(), dv.bfloat16()


def _bounds(layout, S):
    """One list of document lengths per row (the rest of the row is padding) -> int32 [B, S, 2]."""
    b = torch.zeros(len(layout), S, 2, dtype=torch.int32)
    for r, docs in enumerate(layout):
        at = 0
        for n in docs:
            b[r, at:at + n, 0], b[r, at:at + n, 1] = at, at + n
            at += n
        assert at <= S
    return b


S = 384
DOCS = [[1, 2, 61, 136, 64, 120], [200, 129, 1, 40]]          # 1-token documents, tile edges, tail padding
MASKS = {                                                       # name -> (mask, causal)
    "causal": lambda: (_bounds(DOCS, S), True),
    "packed": lambda: (_bounds(DOCS, S), False),
    "windowed": lambda: (window_bounds(_bounds(DOCS, S), 40), False),
    "key_padding": lambda: (torch.tensor([65, S], dtype=torch.int32), False),
}


def _inputs(B, H, Hkv, S, d, seed, family="randn"):
    g = torch.Generator().manual_seed(seed)
    q, dout = (torch.randn(B, H, S, d, generator=g) for _ in range(2))
    k, v = (torch.randn(B, Hkv, S, d, generator=g) for _ in range(2))
    if family == "late_max":                                    # each row's largest scores in its last visible tile
        q[..., 0] = 4.0
        k[..., 0] = torch.linspace(-8.0, 8.0, S)
    return tuple(t.bfloat16() for t in (q, k, v, dout))


def _problem(mask_name, d, family="randn", H=4, Hkv=2, seed=0):
    mask, causal = MASKS[mask_name]()
    if not causal:
        Hkv = H                                                 # the key-padding and document kernels are multi-head
    B = mask.shape[0]
    q, k, v, dout = _inputs(B, H, Hkv, S, d, seed, family)
    return q, k, v, dout, nm.attention_visible(mask, S, causal)


def _check_fwd(q, k, v, vis, o, lse, ref_vis=None):
    ref = nm.attention_reference(q, k, v, vis if ref_vis is None else ref_vis, SCALE[q.shape[-1]])
    return nm.check_attention("fwd", {"o": o, "lse": lse}, ref)


def _check_bwd(q, k, v, o, lse, dout, vis, grads):
    ref = nm.attention_bwd_reference(q, k, v, o, lse, dout, vis, SCALE[q.shape[-1]])
    return nm.check_attention("bwd", dict(zip(("dq", "dk", "dv"), grads)), ref)


@pytest.mark.parametrize("family", ["randn", "late_max"])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("mask_name", sorted(MASKS))
def test_emulated_kernels_stay_well_inside_every_bound(mask_name, d, family):
    q, k, v, dout, vis = _problem(mask_name, d, family)
    o, lse = emulate_fwd(q, k, v, vis)
    worst = _check_fwd(q, k, v, vis, o, lse)
    worst.update(_check_bwd(q, k, v, o, lse, dout, vis, emulate_bwd(q, k, v, o, lse, dout, vis)))
    assert max(worst.values()) <= 0.9, worst
    assert min(worst.values()) > 0.0, worst


def _rejected(fn):
    with pytest.raises(AssertionError, match="out of bound; worst at|-inf where the reference"):
        fn()


def _fwd_fault(mask_name, edit, d=64):
    """Forward with the mask `edit(vis)` returns, checked against the true mask."""
    q, k, v, _, vis = _problem(mask_name, d)
    bad = edit(vis.clone())
    assert not torch.equal(bad, vis)
    o, lse = emulate_fwd(q, k, v, bad)
    _rejected(lambda: _check_fwd(q, k, v, vis, o, lse))
    return q, k, v, vis, o


def _starts(mask_name):
    """(batch row, first position) of every document after the first in its row."""
    mask, _ = MASKS[mask_name]()
    return [(b, i) for b in range(mask.shape[0]) for i in range(1, S) if int(mask[b, i, 0]) == i and mask[b, i, 1] > i]


def test_hidden_causal_diagonal_fails():
    _fwd_fault("causal", lambda vis: vis & ~torch.eye(S, dtype=torch.bool))


def test_one_key_past_the_diagonal_on_rows_63_mod_64_fails():
    def edit(vis):
        for i in range(63, S - 1, 64):
            vis[:, i, i + 1] |= vis[:, i + 1, i]                # the next key, where it is in the same document
        return vis
    _fwd_fault("causal", edit)


def test_first_row_of_a_document_seeing_the_previous_document_fails():
    b, i = _starts("causal")[2]

    def edit(vis):
        vis[b, i, i - 1] = True
        return vis
    _fwd_fault("causal", edit)


def test_key_len_visible_at_len_65_fails():
    def edit(vis):
        vis[0, :, 65] = True
        return vis
    _fwd_fault("key_padding", edit)


def _window_row_fault(vis, b=0, i=130, w=40):
    vis[b, i, i - w - 1] = vis[b, i, i + w + 1] = True          # |i - j| <= w + 1 on row i, inside document 64 .. 199
    return vis


def _row_70_fault(vis, b=0):
    vis[b, 70, 64] = False                                      # row 70 loses its document's first key
    return vis


def test_window_one_wider_on_one_row_fails():
    _fwd_fault("windowed", _window_row_fault)


def test_row_losing_its_documents_first_key_fails():
    _fwd_fault("causal", _row_70_fault)


def test_gqa_reading_the_wrong_kv_head_fails():
    q, k, v, _, vis = _problem("causal", 64)
    o, lse = emulate_fwd(q, k, v, vis, kv_head=[h % k.shape[1] for h in range(q.shape[1])])
    _rejected(lambda: _check_fwd(q, k, v, vis, o, lse))


def test_lse_written_one_row_down_fails():
    q, k, v, _, vis = _problem("causal", 64)
    o, lse = emulate_fwd(q, k, v, vis)
    lse[1, 2, 101] = lse[1, 2, 100]
    _rejected(lambda: _check_fwd(q, k, v, vis, o, lse))


def _bwd_fault(mask_name, d=64, post=None, **fault):
    q, k, v, dout, vis = _problem(mask_name, d)
    o, lse = emulate_fwd(q, k, v, vis)
    grads = list(emulate_bwd(q, k, v, o, lse, dout, vis, **fault))
    if post is not None:
        post(grads)
    _rejected(lambda: _check_bwd(q, k, v, o, lse, dout, vis, grads))


@pytest.mark.parametrize("mask_name", ["causal", "packed"])
def test_dropped_last_query_stage_of_one_key_tile_fails(mask_name):
    _bwd_fault(mask_name, drop_stage=(0, 1))


def test_gqa_dkdv_summing_only_the_first_head_of_each_group_fails():
    _bwd_fault("causal", first_head_only=True)


def test_d_from_the_neighbouring_head_fails():
    _bwd_fault("causal", d_head=[(h + 1) % 4 for h in range(4)])


def test_second_column_chunk_of_one_d128_dv_tile_left_at_zero_fails():
    def post(grads):
        grads[2][1, 1, 128:256, 64:] = 0
    _bwd_fault("causal", d=128, post=post)


# ---- what the older global checks see ----------------------------------------------------------------------------------
OLD_S = 1024
OLD_DOCS = [[1, 2, 61, 300, 660], [200, 129, 1, 54, 640], [OLD_S], [512, 512]]


def _old_checks_pass(o, o_sdpa, ref):
    """rel_err < 1e-2 and the RMS form rms(err) <= 1.5 rms(SDPA err) + 2e-3 rms(ref) of the SDPA-relative tests."""
    def rms(t):
        return float(t.double().pow(2).mean().sqrt())
    return nm.rel_err(o, ref) < 1e-2 and rms(o.double() - ref) <= 1.5 * rms(o_sdpa.double() - ref) + 2e-3 * rms(ref)


@pytest.mark.parametrize("fault", ["window_one_row", "row_70_loses_first_key"])
def test_single_row_mask_faults_pass_the_old_global_checks_but_not_the_bound(fault):
    H = 8
    window = fault == "window_one_row"
    bounds = _bounds(OLD_DOCS, OLD_S)
    if window:
        bounds = window_bounds(bounds, 40)
    vis = nm.attention_visible(bounds, OLD_S, causal=not window)
    q, k, v, _ = _inputs(len(OLD_DOCS), H, H, OLD_S, 64, seed=1)
    bad = vis[:, None].repeat(1, H, 1, 1)                       # the fault is on one row of one head
    (_window_row_fault if window else _row_70_fault)(bad[:, 3])
    o, lse = emulate_fwd(q, k, v, bad)
    ref = nm.attention_reference(q, k, v, vis, SCALE[64])
    sdpa = F.scaled_dot_product_attention(q, k, v, attn_mask=vis[:, None])
    assert _old_checks_pass(o, sdpa, ref["o"][0])
    with pytest.raises(AssertionError, match=r"out of bound; worst at \(0, 3, (130|70), "):
        nm.check_attention("fwd", {"o": o, "lse": lse}, ref)


def test_error_message_names_the_wrong_element():
    q, k, v, _, vis = _problem("causal", 64)
    o, lse = emulate_fwd(q, k, v, vis)
    o[1, 2, 77, 5] += 0.5
    ref = nm.attention_reference(q, k, v, vis, SCALE[64])
    with pytest.raises(AssertionError, match=r"o \[b, h, s, d\]: 1 of \d+ elements out of bound; worst at \(1, 2, 77, 5\)"):
        nm.check_attention("fwd", {"o": o, "lse": lse}, ref)
    lse[0, 1, 0] = -math.inf
    with pytest.raises(AssertionError, match=r"-inf where the reference is not or the reverse; first at \(0, 1, 0\)"):
        nm.check_attention("fwd", {"lse": lse}, ref)
