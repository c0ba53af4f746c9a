"""The argument contract of the CLIP bindings (the ``_C.clip`` namespace of static entry points), exercised with CPU
tensors, and the check that every tensor binding in that namespace has a row here.

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


# "<submodule>.<binding>" -> (builder of well-formed CPU arguments, [(argument named by the error, {position: malformed value})])
ROWS = {
    "clip.quick_gelu_fwd": (lambda: [bf(64)], [("pre", {0: torch.zeros(8, dtype=torch.uint8)}), ("pre", {0: strided(bf(64))})]),
    "clip.quick_gelu_bwd": (lambda: [bf(64), bf(64)],
                            [("pre", {1: torch.zeros(8, dtype=torch.uint8)}), ("dy", {0: f32(64)}), ("dy", {0: bf(32)}),
                             ("dy", {0: strided(bf(64))})]),
    "clip.l2norm_fwd": (lambda: [bf(8, 64)],
                        [("x", {0: f32(8, 64)}), ("x", {0: bf(8, 12)}), ("x", {0: bf(512)}), ("x", {0: strided(bf(8, 64))}),
                         ("x", {0: offset(bf(8, 64))})]),
    "clip.l2norm_bwd": (lambda: [bf(8, 64), bf(8, 64), f32(8)],
                        [("x", {1: bf(8, 12)}), ("du", {0: bf(8, 32)}), ("du", {0: f32(8, 64)}), ("du", {0: offset(bf(8, 64))}),
                         ("rnorm", {2: f32(4)}), ("rnorm", {2: bf(8)})]),
    "clip.contrastive_xent": (lambda: [f32(8, 32), f32(8, 32), f32(1), 8],
                              [("z_img", {0: bf(8, 32)}), ("z_img", {0: f32(8, 4)}), ("z_img", {0: strided(f32(8, 32))}),
                               ("z_txt", {1: f32(8, 16)}), ("logit_scale", {2: f32(2)}), ("logit_scale", {2: bf(1)}),
                               ("label_offset", {3: 25}), ("label_offset", {3: -1})]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_clip_tensor_binding_has_a_row():
    C = _ext.get()
    assert isinstance(C.clip, type)
    found = {f"clip.{k}" for k in dir(C.clip) if not k.startswith("_") and _takes_tensor(getattr(C.clip, k).__doc__)}
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
