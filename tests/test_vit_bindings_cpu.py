"""The argument contract of the Vision Transformer bindings (the ``_C.vit`` submodule), exercised with CPU tensors.

They follow the contract of every other native binding: each tensor argument's dtype, shape, layout and alignment is
checked, then that all of them are CUDA tensors on one device, and only then does the binding allocate or launch.  With
CPU tensors a well-formed call therefore stops at the device check, and a malformed one at the check of the argument it
breaks, with "<binding>: <argument> must be ...".
"""
import re
import types

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
    "vit.patchify": (lambda: [bf(2, 3, 16, 32), 16, 128],
                     [("images", {0: f32(2, 3, 16, 32)}), ("images", {0: bf(2, 3, 16)}), ("images", {0: offset(bf(2, 3, 16, 32))}),
                      ("images", {0: bf(2, 3, 16, 32).permute(0, 1, 3, 2)}), ("patch", {1: 12}), ("patch", {1: 32}),
                      ("tokens", {2: 5})]),
    "vit.patch_assemble": (lambda: [bf(128, 16), bf(1, 1, 16), bf(1, 3, 16), 2],
                           [("y", {0: f32(128, 16)}), ("y", {0: bf(128, 12)}), ("y", {0: offset(bf(128, 16))}),
                            ("class_token", {1: bf(1, 1, 8)}), ("pos_embedding", {2: bf(1, 3, 8)}),
                            ("pos_embedding", {2: strided(bf(1, 3, 16))}), ("batch", {3: 64})]),
    "vit.patch_embed_bwd": (lambda: [bf(128, 16), 2, 3],
                            [("dy", {0: f32(128, 16)}), ("dy", {0: bf(128, 12)}), ("dy", {0: offset(bf(128, 16))}),
                             ("batch", {1: 64}), ("batch", {2: 0})]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_submodule_tensor_binding_has_a_row():
    C = _ext.get()
    found = set()
    for sub in dir(C):
        mod = getattr(C, sub)
        if not isinstance(mod, types.ModuleType):
            continue
        for k in dir(mod):
            f = getattr(mod, k)
            if callable(f) and not isinstance(f, type) and _takes_tensor(f.__doc__):
                found.add(f"{sub}.{k}")
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
