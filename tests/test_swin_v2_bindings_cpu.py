"""The argument contract of Swin V2's cosine window-attention bindings (the ``_C.swin_v2`` namespace of static entry
points), exercised with CPU tensors, and the check that every tensor binding in that namespace has a row here.

They follow the contract of every other native binding: each tensor argument's dtype, shape, layout and alignment is
checked, then that all of them are CUDA tensors on one device, and only then does the binding allocate or launch.  With
CPU tensors a well-formed call therefore stops at the device check, and a malformed one at the check of the argument it
breaks, with "<binding>: <argument> must be ...".
"""
import re

import pytest
import torch

from b200ddp import _ext

pytestmark = pytest.mark.skipif(not _ext.available(), reason="native extension not built")

# Only where no GPU is visible: a check missed by mistake must never hand a host pointer to a kernel on a shared GPU, and
# here the device check is what stops every call before a launch.
if torch.cuda.is_available():
    pytest.skip("binding contracts are exercised on CPU tensors only, on machines without a GPU", allow_module_level=True)

B, H, W, HEADS = 2, 16, 24, 2
ROWS_, C = B * H * W, 32 * HEADS


def bf(*s):
    return torch.zeros(*s, dtype=torch.bfloat16)


def f32(*s):
    return torch.zeros(*s, dtype=torch.float32)


def strided(t):
    """A non-contiguous view with t's shape and dtype."""
    return torch.zeros(*t.shape, 2, dtype=t.dtype)[..., 0]


def offset(t, elems=1):
    """A contiguous view with t's shape and dtype whose address is `elems` elements past an allocation's start."""
    return torch.zeros(t.numel() + elems, dtype=t.dtype)[elems:].view(t.shape)


GEOMETRY = [B, H, W, 4, 4]
BAD_QKV = [f32(ROWS_, 3 * C), bf(ROWS_, 3 * 64 * HEADS), bf(ROWS_ + 8, 3 * C), bf(ROWS_ * 3 * C), strided(bf(ROWS_, 3 * C)),
           offset(bf(ROWS_, 3 * C))]
BAD_TABLE = [bf(225, HEADS), f32(169, HEADS), f32(225, 0), f32(225 * HEADS), strided(f32(225, HEADS))]
BAD_SCALE = [bf(HEADS), f32(HEADS + 1), f32(HEADS, 1), strided(f32(HEADS))]
BAD_GEOMETRY = [[0, H, W, 4, 4], [B, 12, W, 4, 4], [B, H, 20, 4, 4], [B, 0, W, 4, 4], [B, H, W, 8, 4], [B, H, W, 4, -1],
                [B, 14, 14, 3, 3], [70000, H, W, 4, 4]]


def _common(q, t, g0):
    """Rows for the qkv at position q, the table at t, the scale at t + 1 and the geometry starting at g0."""
    return ([("qkv", {q: v}) for v in BAD_QKV] + [("table", {t: v}) for v in BAD_TABLE] + [("scale", {t + 1: v}) for v in BAD_SCALE] +
            [("geometry", dict(enumerate(g, g0))) for g in BAD_GEOMETRY])


# "<namespace>.<binding>" -> (builder of well-formed CPU arguments, [(argument named by the error, {position: malformed value})])
ROWS = {
    "swin_v2.attention_fwd": (lambda: [bf(ROWS_, 3 * C), f32(225, HEADS), f32(HEADS), *GEOMETRY], _common(0, 1, 3)),
    "swin_v2.attention_bwd": (lambda: [bf(ROWS_, C), bf(ROWS_, 3 * C), bf(ROWS_, C), f32(ROWS_, HEADS), f32(225, HEADS), f32(HEADS),
                                       *GEOMETRY],
                              _common(1, 4, 6) +
                              [("dout", {0: v}) for v in (f32(ROWS_, C), bf(ROWS_, C + 32), strided(bf(ROWS_, C)), offset(bf(ROWS_, C)))] +
                              [("o", {2: v}) for v in (f32(ROWS_, C), bf(ROWS_ - 1, C), strided(bf(ROWS_, C)), offset(bf(ROWS_, C)))] +
                              [("lse", {3: v}) for v in (bf(ROWS_, HEADS), f32(ROWS_, HEADS + 1), f32(HEADS, ROWS_).t())]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_swin_v2_tensor_binding_has_a_row():
    C_ = _ext.get()
    assert isinstance(C_.swin_v2, type)
    found = {f"swin_v2.{k}" for k in dir(C_.swin_v2) if not k.startswith("_") and _takes_tensor(getattr(C_.swin_v2, k).__doc__)}
    assert found == set(ROWS)


@pytest.mark.parametrize("name", sorted(ROWS))
def test_well_formed_call_reaches_the_device_check(name):
    build, _ = ROWS[name]
    fn = name.split(".")[1]
    with pytest.raises(RuntimeError, match=rf"^{fn}: \w+ must be a CUDA tensor, got cpu"):
        _binding(name)(*build())


@pytest.mark.parametrize("name,arg,change", [(n, a, c) for n in sorted(ROWS) for a, c in ROWS[n][1]],
                         ids=lambda v: v if isinstance(v, str) else "")
def test_malformed_argument_is_rejected(name, arg, change):
    args = ROWS[name][0]()
    for pos, value in change.items():
        args[pos] = value
    fn = name.split(".")[1]
    with pytest.raises(RuntimeError, match=rf"^{re.escape(fn)}: {arg} must be ") as info:
        _binding(name)(*args)
    assert "CUDA tensor" not in str(info.value)


def test_messages_name_the_window_and_head_dim():
    fwd = _binding("swin_v2.attention_fwd")
    with pytest.raises(RuntimeError, match="multiples of 8"):
        fwd(bf(ROWS_, 3 * C), f32(225, HEADS), f32(HEADS), B, 12, W, 4, 4)
    with pytest.raises(RuntimeError, match="head dim 32"):
        fwd(bf(ROWS_, 3 * 64 * HEADS), f32(225, HEADS), f32(HEADS), *GEOMETRY)
