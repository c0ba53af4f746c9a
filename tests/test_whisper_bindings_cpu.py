"""The argument contract of Whisper's log-mel and stem bindings (the ``_C.whisper`` namespace of static entry points),
exercised with CPU tensors, and the check that every tensor binding in that namespace has a row here.

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

B, T, S, D = 2, 128, 128, 64


def bf(*s):
    return torch.zeros(*s, dtype=torch.bfloat16)


def f32(*s):
    return torch.zeros(*s, dtype=torch.float32)


def i16(*s):
    return torch.zeros(*s, dtype=torch.int16)


def strided(t):
    """A view with t's shape and dtype whose last dimension's elements are two apart."""
    return torch.zeros(*t.shape, 2, dtype=t.dtype)[..., 0]


def offset(t, elems=1):
    """A contiguous view with t's shape and dtype whose address is `elems` elements past an allocation's start."""
    return torch.zeros(t.numel() + elems, dtype=t.dtype)[elems:].view(t.shape)


# "<namespace>.<binding>" -> (builder of well-formed CPU arguments, [(argument named by the error, {position: malformed value})])
ROWS = {
    "whisper.log_mel": (lambda: [i16(B, 480000), f32(201, 80), True],
                        [("wave", {0: v}) for v in (f32(B, 480000), torch.zeros(B, 480000, dtype=torch.int32), i16(B, 479999), i16(480000),
                                                    strided(i16(B, 480000)), i16(0, 480000))] +
                        [("filters", {1: v}) for v in (bf(201, 80), f32(80, 201), strided(f32(201, 80)))] +
                        [("out", {3: v}) for v in (f32(B, 80, 3000), bf(B, 80, 2999), strided(bf(B, 80, 3000)))]),
    "whisper.mel_patches": (lambda: [bf(B, 80, T)],
                            [("features", {0: v}) for v in (f32(B, 80, T), bf(B, 81, T), bf(B * 80, T), strided(bf(B, 80, T)), bf(0, 80, T))]),
    "whisper.frame_patches": (lambda: [bf(B * T, D), T, S],
                              [("h1", {0: v}) for v in (f32(B * T, D), bf(B * T + 1, D), bf(B * T, D + 4), strided(bf(B * T, D)),
                                                        offset(bf(B * T, D)), bf(B * T))] +
                              [("frames", {1: v}) for v in (T + 1, 0)] + [("frames", {2: T // 2 - 1})]),
    "whisper.frame_patches_bwd": (lambda: [bf(B * S, 3 * D), T, S],
                                  [("dp2", {0: v}) for v in (f32(B * S, 3 * D), bf(B * S + 1, 3 * D), bf(B * S, 3 * D + 1),
                                                             bf(B * S, 3 * D + 12), strided(bf(B * S, 3 * D)), offset(bf(B * S, 3 * D)))] +
                                  [("frames", {1: v}) for v in (T - 1, -2)] + [("frames", {2: T // 2 - 1})]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_whisper_tensor_binding_has_a_row():
    C_ = _ext.get()
    assert isinstance(C_.whisper, type)
    found = {f"whisper.{k}" for k in dir(C_.whisper) if not k.startswith("_") and _takes_tensor(getattr(C_.whisper, k).__doc__)}
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
        if pos == len(args):
            args.append(value)
        else:
            args[pos] = value
    fn = name.split(".")[1]
    with pytest.raises(RuntimeError, match=rf"^{re.escape(fn)}: {arg} must be ") as info:
        _binding(name)(*args)
    assert "CUDA tensor" not in str(info.value)
