"""The argument contract of Mamba-2's conv, SSD and gated-norm bindings (the ``_C.mamba2`` namespace of static entry
points), exercised with CPU tensors, and the check that every tensor binding in that namespace has a row here.

They follow the contract of every other native binding: each tensor argument's dtype, shape, layout and alignment is
checked, then that all of them are CUDA tensors on one device, and only then does the binding allocate or launch.  With
CPU tensors a well-formed call therefore stops at the device check, and a malformed one at the check of the argument it
breaks, with "<binding>: <argument> must be ...".  Row views (x, dx_out, dt, ddt_out, z, dz_out) are column windows of a
wider row, as Mamba-2 reads them from in_proj's output.
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

B, S, H = 2, 37, 8
T, E, N = B * S, 64 * H, 128
CD = E + 2 * N                    # conv_dim
W = 2 * E + 2 * N + H             # in_proj's output width
NE = 1536                         # the gated norm's width (the wide kernels take 1024 < E <= 4096)


def bf(*s):
    return torch.zeros(*s, dtype=torch.bfloat16)


def f32(*s):
    return torch.zeros(*s, dtype=torch.float32)


def i32(*s):
    return torch.zeros(*s, dtype=torch.int32)


def strided(t):
    """A view with t's shape and dtype whose columns are two elements apart."""
    return torch.zeros(*t.shape, 2, dtype=t.dtype)[..., 0]


def offset(t, elems=1):
    """A contiguous view with t's shape and dtype whose address is `elems` elements past an allocation's start."""
    return torch.zeros(t.numel() + elems, dtype=t.dtype)[elems:].view(t.shape)


def window(rows, width, col, cols, dtype=torch.bfloat16):
    """Columns [col, col + cols) of a [rows, width] tensor."""
    return torch.zeros(rows, width, dtype=dtype)[:, col:col + cols]


BAD_BOUNDS = [f32(B, S, 2), i32(B, S, 3), i32(B * S, 2), strided(i32(B, S, 2)), offset(i32(B, S, 2)), i32(0, S, 2)]


def _bad_view(rows, cols):
    """Malformed row views: wrong dtype, rows, column stride, alignment, and a pitch that is not a multiple of 8."""
    return [window(rows, W, 0, cols, torch.float32), window(rows + 1, W, 0, cols), strided(bf(rows, cols)), offset(bf(rows, cols)),
            window(rows, cols + 4, 0, cols)]


def _conv_args():
    return [window(T, W, E, CD), f32(CD, 4), f32(CD), i32(B, S, 2)]


def _ssd_args():
    return [bf(T, CD), window(T, W, W - H, H), f32(H), f32(H), f32(H), i32(B, S, 2)]


def _ssd_rows(first):
    xbc, dt, a, d, b, bounds = range(first, first + 6)
    return ([("bounds", {bounds: v}) for v in BAD_BOUNDS] +
            [("xbc", {xbc: v}) for v in (f32(T, CD), bf(T + 1, CD), bf(T, CD + 8), bf(T, 256 + 64 * 4), strided(bf(T, CD)),
                                         offset(bf(T, CD)))] +
            [("dt", {dt: v}) for v in _bad_view(T, H) + [bf(T, H + 1)]] +
            [("A_log", {a: v}) for v in (bf(H), f32(H + 1))] + [("D", {d: v}) for v in (bf(H), f32(H, 1))] +
            [("dt_bias", {b: v}) for v in (f32(H - 1),)])


def _norm_args():
    return [bf(T, NE), window(T, 3352, 0, NE), bf(NE), 1e-5]


# "<namespace>.<binding>" -> (builder of well-formed CPU arguments, [(argument named by the error, {position: malformed value})])
ROWS = {
    "mamba2.conv_fwd": (_conv_args,
                        [("bounds", {3: v}) for v in BAD_BOUNDS] +
                        [("x", {0: v}) for v in _bad_view(T, CD) + [window(T, W, E, CD - 4)]] +
                        [("weight", {1: v}) for v in (bf(CD, 4), f32(CD, 3), offset(f32(CD, 4)))] +
                        [("bias", {2: v}) for v in (bf(CD), f32(CD + 8))]),
    "mamba2.conv_bwd": (lambda: [bf(T, CD)] + _conv_args() + [window(T, W, E, CD)],
                        [("bounds", {4: v}) for v in BAD_BOUNDS] + [("x", {1: v}) for v in _bad_view(T, CD)] +
                        [("du", {0: v}) for v in (f32(T, CD), bf(T, CD + 8), offset(bf(T, CD)))] +
                        [("weight", {2: v}) for v in (bf(CD, 4), f32(CD, 5))] + [("bias", {3: v}) for v in (f32(CD - 8),)] +
                        [("dx_out", {5: v}) for v in _bad_view(T, CD)]),
    "mamba2.ssd_fwd": (_ssd_args, _ssd_rows(0)),
    "mamba2.ssd_bwd": (lambda: [bf(T, E)] + _ssd_args() + [window(T, W, W - H, H)],
                       _ssd_rows(1) + [("dy", {0: v}) for v in (f32(T, E), bf(T, E + 8), strided(bf(T, E)))] +
                       [("ddt_out", {7: v}) for v in _bad_view(T, H)]),
    "mamba2.gated_norm_fwd": (_norm_args,
                              [("y", {0: v}) for v in (f32(T, NE), bf(T, 1024), bf(T, NE + 4), strided(bf(T, NE)), bf(0, NE))] +
                              [("z", {1: v}) for v in _bad_view(T, NE)] +
                              [("weight", {2: v}) for v in (f32(NE), bf(NE + 8), offset(bf(NE)))]),
    "mamba2.gated_norm_bwd": (lambda: [bf(T, NE)] + _norm_args()[:3] + [f32(T), window(T, 3352, 0, NE)],
                              [("y", {1: v}) for v in (f32(T, NE), bf(T, 4104))] +
                              [("dout", {0: v}) for v in (f32(T, NE), bf(T, NE + 8), offset(bf(T, NE)))] +
                              [("z", {2: v}) for v in _bad_view(T, NE)] + [("weight", {3: v}) for v in (f32(NE),)] +
                              [("rstd", {4: v}) for v in (bf(T), f32(T + 1))] + [("dz_out", {5: v}) for v in _bad_view(T, NE)]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_mamba2_tensor_binding_has_a_row():
    C_ = _ext.get()
    assert isinstance(C_.mamba2, type)
    found = {f"mamba2.{k}" for k in dir(C_.mamba2) if not k.startswith("_") and _takes_tensor(getattr(C_.mamba2, k).__doc__)}
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
