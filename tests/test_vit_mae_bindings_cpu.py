"""The argument contract of the masked-autoencoder bindings (the ``_C.mae`` namespace of static entry points), exercised
with CPU tensors, and the check that every tensor binding in that namespace has a row here.  A well-formed call stops at
the device check; a malformed one at the check of the argument it breaks, with "<binding>: <argument> must be ..."."""
import re

import pytest
import torch

from b200ddp import _ext

pytestmark = pytest.mark.skipif(not _ext.available(), reason="native extension not built")

# Only where no GPU is visible: the device check is what stops every call before a launch.
if torch.cuda.is_available():
    pytest.skip("binding contracts are exercised on CPU tensors only, on machines without a GPU", allow_module_level=True)

B, N, K, D, E, H = 2, 196, 49, 64, 64, 2
TE, TD = 128, 512


def bf(*s):
    return torch.zeros(*s, dtype=torch.bfloat16)


def f32(*s):
    return torch.zeros(*s, dtype=torch.float32)


def i32(*s):
    return torch.zeros(*s, dtype=torch.int32)


def strided(t):
    return torch.zeros(*t.shape, 2, dtype=t.dtype)[..., 0]


def offset(t, elems=1):
    return torch.zeros(t.numel() + elems, dtype=t.dtype)[elems:].view(t.shape)


def img(*s):
    return bf(*s) if s else bf(B, 3, 224, 224)


ROWS = {
    "mae.shuffle": (lambda: [f32(B, N), K],
                    [("noise", {0: v}) for v in (bf(B, N), f32(B, 1025), f32(N), strided(f32(B, N)), f32(0, N))] +
                    [("keep", {1: v}) for v in (-1, N + 1)]),
    "mae.patchify": (lambda: [img(), i32(B, K), 16, TE],
                     [("images", {0: v}) for v in (f32(B, 3, 224, 224), bf(B, 3, 224), strided(img()), offset(img()))] +
                     [("patch", {2: v}) for v in (12, 7, 0)] +
                     [("ids_keep", {1: v}) for v in (torch.zeros(B, K, dtype=torch.long), i32(B + 1, K), i32(B, N + 1))] +
                     [("tokens", {3: v}) for v in (B * (K + 1) - 1,)]),
    "mae.patch_assemble": (lambda: [bf(TE, D), bf(1, 1, D), bf(1, N + 1, D), i32(B, K)],
                           [("y", {0: v}) for v in (f32(TE, D), bf(TE, D + 4), bf(TE * D), offset(bf(TE, D)))] +
                           [("class_token", {1: v}) for v in (bf(1, 1, D + 8), f32(1, 1, D))] +
                           [("pos_embedding", {2: v}) for v in (bf(1, N + 1, D + 8), f32(1, N + 1, D))] +
                           [("ids_keep", {3: v}) for v in (torch.zeros(B, K, dtype=torch.long), i32(B, N + 1), i32(3, K))]),
    "mae.patch_embed_bwd": (lambda: [bf(TE, D), B, K + 1],
                            [("dy", {0: v}) for v in (f32(TE, D), bf(TE, D + 4), offset(bf(TE, D)), bf(TE))] +
                            [("batch", {1: v}) for v in (0, 3)]),
    "mae.unshuffle": (lambda: [bf(TE, E), bf(1, 1, E), bf(1, N + 1, E), i32(B, N), K, TD],
                      [("y", {0: v}) for v in (f32(TE, E), bf(TE, E + 4), bf(TE, 4096), offset(bf(TE, E)), bf(B * (K + 1) - 1, E))] +
                      [("mask_token", {1: v}) for v in (bf(1, 1, E + 8), f32(1, 1, E))] +
                      [("pos_embedding", {2: v}) for v in (bf(1, N, E), f32(1, N + 1, E))] +
                      [("ids_restore", {3: v}) for v in (torch.zeros(B, N, dtype=torch.long), i32(B, 1025), i32(0, N))] +
                      [("keep", {4: v}) for v in (-1, N + 1)] + [("rows", {5: B * (N + 1) - 1})]),
    "mae.unshuffle_bwd": (lambda: [bf(TD, E), i32(B, K), i32(B, N), TE],
                          [("dz", {0: v}) for v in (f32(TD, E), bf(TD, E + 4), offset(bf(TD, E)), bf(B * (N + 1) - 1, E))] +
                          [("ids_keep", {1: v}) for v in (torch.zeros(B, K, dtype=torch.long), i32(0, K))] + [("keep", {1: i32(B, N + 1)})] +
                          [("ids_restore", {2: v}) for v in (i32(B + 1, N), torch.zeros(B, N, dtype=torch.long))] +
                          [("rows", {3: B * (K + 1) - 1})]),
    "mae.attention_fwd": (lambda: [bf(TD, 96 * H), B, 197],
                          [("qkv", {0: v}) for v in (f32(TD, 96 * H), bf(TD, 96 * H + 8), offset(bf(TD, 96 * H)), strided(bf(TD, 96 * H)))] +
                          [("geometry", {2: v}) for v in (0, 257)] + [("geometry", {1: v}) for v in (0, 3)]),
    "mae.attention_bwd": (lambda: [bf(TD, 32 * H), bf(TD, 96 * H), bf(TD, 32 * H), f32(TD, H), B, 197],
                          [("dout", {0: v}) for v in (f32(TD, 32 * H), bf(TD, 32 * H + 8), offset(bf(TD, 32 * H)))] +
                          [("qkv", {1: v}) for v in (f32(TD, 96 * H), bf(TD, 100))] +
                          [("o", {2: v}) for v in (bf(TD - 1, 32 * H),)] + [("lse", {3: v}) for v in (f32(TD, H + 1), bf(TD, H))] +
                          [("geometry", {5: 300})]),
    "mae.loss": (lambda: [bf(TD, 768), img(), i32(B, N), K, False],
                 [("pred", {0: v}) for v in (f32(TD, 768), bf(TD, 770), bf(TD, 1536), offset(bf(TD, 768)), bf(B * (N + 1) - 1, 768))] +
                 [("images", {1: v}) for v in (f32(B, 3, 224, 224), strided(img()))] + [("patch", {1: img(B, 3, 224, 232)})] +
                 [("ids_restore", {2: v}) for v in (i32(B, N - 1), torch.zeros(B, N, dtype=torch.long))] +
                 [("keep", {3: v}) for v in (N, -1)]),
    "mae.loss_bwd": (lambda: [f32(1), bf(TD, 768), img(), i32(B, N), K, True],
                     [("dloss", {0: v}) for v in (f32(2), bf(1))] +
                     [("pred", {1: v}) for v in (f32(TD, 768), offset(bf(TD, 768)))] +
                     [("images", {2: v}) for v in (f32(B, 3, 224, 224),)] +
                     [("ids_restore", {3: v}) for v in (i32(B + 1, N),)] + [("keep", {4: N})]),
}


def _binding(name):
    sub, fn = name.split(".")
    return getattr(getattr(_ext.get(), sub), fn)


def _takes_tensor(doc):
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_mae_tensor_binding_has_a_row():
    C_ = _ext.get()
    assert isinstance(C_.mae, type)
    found = {f"mae.{k}" for k in dir(C_.mae) if not k.startswith("_") and _takes_tensor(getattr(C_.mae, k).__doc__)}
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
