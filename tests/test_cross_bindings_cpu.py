"""The argument contract of the cross-attention bindings (the ``_C.cross`` namespace of static entry points), exercised
with CPU tensors, and the check that every tensor binding in that namespace has a row here.

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

B, SQ, SK, H = 2, 128, 256, 2
HID = H * 64


def bf(*s):
    return torch.zeros(*s, dtype=torch.bfloat16)


def f32(*s):
    return torch.zeros(*s, dtype=torch.float32)


def i32(*s):
    return torch.zeros(*s, dtype=torch.int32)


def strided(t):
    """A non-contiguous view with t's shape and dtype."""
    return torch.zeros(*t.shape, 2, dtype=t.dtype)[..., 0]


def offset(t, elems=1):
    """A contiguous view with t's shape and dtype whose address is `elems` elements past an allocation's start."""
    return torch.zeros(t.numel() + elems, dtype=t.dtype)[elems:].view(t.shape)


def _fwd_args():
    return [bf(B * SQ, HID), bf(B * SK, 2 * HID), i32(B, SQ, 2), H]


def _bwd_args():
    return [bf(B * SQ, HID), bf(B * SQ, HID), bf(B * SK, 2 * HID), bf(B * SQ, HID), f32(B, H, SQ), i32(B, SQ, 2), i32(B, SK, 2), H]


# "<namespace>.<binding>" -> (builder of well-formed CPU arguments, [(argument named by the error, {position: malformed value})])
ROWS = {
    "cross.cross_attention_fwd": (_fwd_args,
                                  [("q", {0: f32(B * SQ, HID)}), ("q", {0: bf(B * SQ, HID + 64)}), ("q", {0: bf(B * SQ + 128, HID)}),
                                   ("q", {0: strided(bf(B * SQ, HID))}), ("q", {0: offset(bf(B * SQ, HID))}),
                                   ("kv", {1: bf(B * SK, HID)}), ("kv", {1: f32(B * SK, 2 * HID)}), ("kv", {1: bf(B * SK + 1, 2 * HID)}),
                                   ("kv", {1: offset(bf(B * SK, 2 * HID))}), ("q_bounds", {2: i32(B, SQ)}),
                                   ("q_bounds", {2: torch.zeros(B, SQ, 2, dtype=torch.int64)}), ("q_bounds", {2: strided(i32(B, SQ, 2))}),
                                   ("q_bounds", {2: i32(0, SQ, 2)}), ("heads", {3: 0})]),
    "cross.cross_attention_bwd": (_bwd_args,
                                  [("dout", {0: f32(B * SQ, HID)}), ("dout", {0: bf(B * SQ, HID - 64)}), ("dout", {0: offset(bf(B * SQ, HID))}),
                                   ("q", {1: bf(B * SQ, HID + 64)}), ("kv", {2: bf(B * SK, HID)}), ("o", {3: bf(B * SQ, HID - 64)}),
                                   ("o", {3: strided(bf(B * SQ, HID))}), ("lse", {4: f32(B, H, SK)}), ("lse", {4: bf(B, H, SQ)}),
                                   ("q_bounds", {5: i32(B, SQ, 3)}), ("kv_bounds", {6: i32(B, SQ, 2)}),
                                   ("kv_bounds", {6: torch.zeros(B, SK, 2, dtype=torch.int64)}), ("kv_bounds", {6: strided(i32(B, SK, 2))}),
                                   ("heads", {7: -1})]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_cross_tensor_binding_has_a_row():
    C = _ext.get()
    assert isinstance(C.cross, type)
    found = {f"cross.{k}" for k in dir(C.cross) if not k.startswith("_") and _takes_tensor(getattr(C.cross, k).__doc__)}
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
