"""The argument contract of Mamba's conv and scan bindings (the ``_C.mamba`` namespace of static entry points), exercised
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

B, S, E, R = 2, 37, 16, 8
T, NC = B * S, 1


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


BAD_BOUNDS = [f32(B, S, 2), i32(B, S, 3), i32(B * S, 2), strided(i32(B, S, 2)), offset(i32(B, S, 2)), i32(0, S, 2)]
BAD_XZ = [f32(T, 2 * E), bf(T + 1, 2 * E), bf(T, 2 * E + 8), bf(T, 8), strided(bf(T, 2 * E)), offset(bf(T, 2 * E))]


def _common(bounds_pos, xz_pos):
    return [("bounds", {bounds_pos: v}) for v in BAD_BOUNDS] + [("xz", {xz_pos: v}) for v in BAD_XZ]


def _scan_rows(first):
    """Rows for u, draw, xbc, A_log, D and dt_bias at positions first .. first + 5 (xz and bounds come between)."""
    u, dr, xbc, a, d, b = first, first + 1, first + 2, first + 4, first + 5, first + 6
    return ([("u", {u: v}) for v in (f32(T, E), bf(T, E + 8), strided(bf(T, E)))] +
            [("draw", {dr: v}) for v in (f32(T, E), bf(T - 1, E))] +
            [("xbc", {xbc: v}) for v in (f32(T, R + 32), bf(T, 31), strided(bf(T, R + 32)))] +
            [("A_log", {a: v}) for v in (bf(E, 16), f32(E, 8))] + [("D", {d: v}) for v in (bf(E), f32(E + 1))] +
            [("dt_bias", {b: v}) for v in (bf(E), f32(E, 1))])


def _scan_args():
    return [bf(T, E), bf(T, E), bf(T, R + 32), bf(T, 2 * E), f32(E, 16), f32(E), f32(E), i32(B, S, 2)]


# "<namespace>.<binding>" -> (builder of well-formed CPU arguments, [(argument named by the error, {position: malformed value})])
ROWS = {
    "mamba.conv_fwd": (lambda: [bf(T, 2 * E), f32(E, 4), f32(E), i32(B, S, 2)],
                       _common(3, 0) + [("weight", {1: v}) for v in (bf(E, 4), f32(E, 3), offset(f32(E, 4)))] +
                       [("bias", {2: v}) for v in (bf(E), f32(E + 8))]),
    "mamba.conv_bwd": (lambda: [bf(T, E), bf(T, 2 * E), f32(E, 4), f32(E), i32(B, S, 2), None],
                       _common(4, 1) + [("du", {0: v}) for v in (f32(T, E), bf(T, E + 8), offset(bf(T, E)))] +
                       [("weight", {2: v}) for v in (bf(E, 4), f32(E, 5))] + [("bias", {3: v}) for v in (f32(E - 8),)] +
                       [("dxz_out", {5: v}) for v in (f32(T, 2 * E), bf(T, E), strided(bf(T, 2 * E)), offset(bf(T, 2 * E)))]),
    "mamba.scan_fwd": (_scan_args, _common(7, 3) + _scan_rows(0)),
    "mamba.scan_bwd": (lambda: [bf(T, E)] + _scan_args() + [f32(B, NC, E, 16), f32(B, NC, E)],
                       _common(8, 4) + _scan_rows(1) + [("dy", {0: v}) for v in (f32(T, E), bf(T, 2 * E))] +
                       [("hstart", {9: v}) for v in (f32(B, 2, E, 16), bf(B, NC, E, 16))] +
                       [("sumd", {10: v}) for v in (f32(B, NC, E + 1), bf(B, NC, E))]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_mamba_tensor_binding_has_a_row():
    C_ = _ext.get()
    assert isinstance(C_.mamba, type)
    found = {f"mamba.{k}" for k in dir(C_.mamba) if not k.startswith("_") and _takes_tensor(getattr(C_.mamba, k).__doc__)}
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
