"""The argument contract of T5's relative-bias bindings (the ``_C.t5`` namespace of static entry points), exercised with
CPU tensors, and the check that every tensor binding in that namespace has a row here.

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

B, S, H = 2, 128, 3
W = 3 * H * 64


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
    return [bf(B * S, W), i32(B, S, 2), f32(H, 257), H, False]


def _bwd_args():
    return [bf(B * S, H * 64), bf(B * S, W), bf(B * S, H * 64), f32(B, H, S), i32(B, S, 2), f32(H, 257), H, True]


# "<namespace>.<binding>" -> (builder of well-formed CPU arguments, [(argument named by the error, {position: malformed value})])
ROWS = {
    "t5.relative_attention_fwd": (_fwd_args,
                                  [("qkv", {0: f32(B * S, W)}), ("qkv", {0: bf(B * S, W + 64)}), ("qkv", {0: bf(B * S + 128, W)}),
                                   ("qkv", {0: strided(bf(B * S, W))}), ("qkv", {0: offset(bf(B * S, W))}),
                                   ("bounds", {1: i32(B, S)}), ("bounds", {1: torch.zeros(B, S, 2, dtype=torch.int64)}),
                                   ("bounds", {1: strided(i32(B, S, 2))}), ("table", {2: f32(H, 256)}), ("table", {2: bf(H, 257)}),
                                   ("table", {2: f32(H + 1, 257)}), ("table", {2: strided(f32(H, 257))}), ("heads", {3: 0})]),
    "t5.relative_attention_bwd": (_bwd_args,
                                  [("dout", {0: f32(B * S, H * 64)}), ("dout", {0: bf(B * S, H * 64 - 64)}),
                                   ("dout", {0: offset(bf(B * S, H * 64))}), ("qkv", {1: bf(B * S, W - 64)}),
                                   ("o", {2: bf(B * S, H * 64 + 64)}), ("o", {2: strided(bf(B * S, H * 64))}),
                                   ("lse", {3: f32(B, H, S + 1)}), ("lse", {3: bf(B, H, S)}), ("bounds", {4: i32(B, S, 3)}),
                                   ("table", {5: f32(257, H)}), ("heads", {6: -1})]),
    "t5.relative_table_fwd": (lambda: [f32(32, H), i32(257)],
                              [("weight", {0: torch.zeros(32, H, dtype=torch.float16)}), ("weight", {0: f32(32 * H)}),
                               ("weight", {0: f32(0, H)}), ("weight", {0: strided(f32(32, H))}), ("bucket", {1: i32(256)}),
                               ("bucket", {1: torch.zeros(257, dtype=torch.int64)})]),
    "t5.relative_table_bwd": (lambda: [f32(H, 257), i32(257), bf(32, H)],
                              [("dtable", {0: f32(H + 1, 257)}), ("dtable", {0: bf(H, 257)}), ("dtable", {0: strided(f32(H, 257))}),
                               ("bucket", {1: i32(257, 1)}), ("weight", {2: torch.zeros(32, H, dtype=torch.float16)}),
                               ("weight", {2: bf(32, H, 1)}), ("weight", {2: bf(32, 0)})]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_t5_tensor_binding_has_a_row():
    C = _ext.get()
    assert isinstance(C.t5, type)
    found = {f"t5.{k}" for k in dir(C.t5) if not k.startswith("_") and _takes_tensor(getattr(C.t5, k).__doc__)}
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
