"""The argument contract of ConvNeXt's depthwise-convolution bindings (the ``_C.convnext`` namespace of static entry
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

B, H, W, C = 2, 9, 13, 16


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


def _act(c=C):
    return bf(B, H, W, c)


# malformed activations, for whichever argument carries the [B, H, W, C] shape
BAD_ACT = [f32(B, H, W, C), bf(B, H, W * C), bf(B, H, W, 12), bf(B, H, W, 4), bf(B, H, W, 1032), bf(0, H, W, C), bf(B, 0, W, C),
           strided(_act()), offset(_act()), bf(B, H, W, C).permute(0, 2, 1, 3)]

# "<namespace>.<binding>" -> (builder of well-formed CPU arguments, [(argument named by the error, {position: malformed value})])
ROWS = {
    "convnext.dwconv_fwd": (lambda: [_act(), bf(C, 49), bf(C)],
                            [("x", {0: t}) for t in BAD_ACT] +
                            [("weight", {1: bf(C, 1, 7, 7)}), ("weight", {1: bf(C + 8, 49)}), ("weight", {1: f32(C, 49)}),
                             ("weight", {1: strided(bf(C, 49))}), ("bias", {2: bf(C + 8)}), ("bias", {2: f32(C)}),
                             ("bias", {2: strided(bf(C))})]),
    "convnext.dwconv_dgrad": (lambda: [_act(), bf(C, 49)],
                              [("dy", {0: t}) for t in BAD_ACT] +
                              [("weight", {1: bf(C, 48)}), ("weight", {1: f32(C, 49)}), ("weight", {1: strided(bf(C, 49))})]),
    "convnext.dwconv_wgrad": (lambda: [_act(), _act()],
                              [("x", {1: t}) for t in BAD_ACT] +
                              [("dy", {0: f32(B, H, W, C)}), ("dy", {0: bf(B, H + 1, W, C)}), ("dy", {0: bf(B, H, W, C + 8)}),
                               ("dy", {0: strided(_act())}), ("dy", {0: offset(_act())})]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_convnext_tensor_binding_has_a_row():
    C_ = _ext.get()
    assert isinstance(C_.convnext, type)
    found = {f"convnext.{k}" for k in dir(C_.convnext) if not k.startswith("_") and _takes_tensor(getattr(C_.convnext, k).__doc__)}
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
