"""The argument contract of the native bindings, exercised with CPU tensors.

Every binding that takes a tensor checks each tensor argument's dtype, shape, layout and alignment, then that all of them
are CUDA tensors on one device, and only then allocates or launches.  With CPU tensors a well-formed call therefore stops
at the device check, and a malformed one at the check of the argument it breaks, with "<binding>: <argument> ...".
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

# Bindings that also take a PeerArena, which cannot be built without a GPU.
EXEMPT = {"allreduce_tensors", "broadcast_tensors", "peer_pull", "peer_push"}


def bf(*s):
    return torch.zeros(*s, dtype=torch.bfloat16)


def f32(*s):
    return torch.zeros(*s, dtype=torch.float32)


def i32(*s):
    return torch.zeros(*s, dtype=torch.int32)


def i64(*s):
    return torch.zeros(*s, dtype=torch.int64)


def u8(*s):
    return torch.zeros(*s, dtype=torch.uint8)


def e4m3(*s):
    return torch.zeros(*s, dtype=torch.float8_e4m3fn)


def cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def strided(t):
    """A non-contiguous view with t's shape and dtype."""
    return torch.zeros(*t.shape, 2, dtype=t.dtype)[..., 0]


def offset(t, elems=1):
    """A contiguous view with t's shape and dtype whose address is `elems` elements past an allocation's start."""
    return torch.zeros(t.numel() + elems, dtype=t.dtype)[elems:].view(t.shape)


# qkv for one sequence of 128 rows: multi-head (1 head), grouped-query (2 query heads, 1 key/value head), head dim 128
QKV, QKV_GQA, QKV_128 = (lambda: bf(128, 192)), (lambda: bf(128, 256)), (lambda: bf(128, 384))
BOUNDS = lambda: i32(1, 128, 2)  # noqa: E731


def attn_rows(mask, mask_name, heads, kv_heads, cols, hd):
    """Forward and backward rows of one attention mode."""
    kv = () if kv_heads is None else (kv_heads,)
    o_cols = heads * hd
    fwd = (lambda: [bf(128, cols), mask(), heads, *kv, None, None],
           [("qkv", {0: bf(128, cols + 64)}), ("qkv", {0: f32(128, cols)}), ("qkv", {0: offset(bf(128, cols))}),
            ("qkv", {0: strided(bf(128, cols))}), (mask_name, {1: i64(*mask().shape)}),
            ("o", {3 + len(kv): bf(128, o_cols + 8)}), ("o", {3 + len(kv): offset(bf(128, o_cols))}),
            ("lse", {4 + len(kv): f32(1, heads, 64)}), ("lse", {4 + len(kv): bf(1, heads, 128)})])
    bwd = (lambda: [bf(128, o_cols), bf(128, cols), bf(128, o_cols), f32(1, heads, 128), mask(), heads, *kv, None],
           [("dout", {0: bf(128, o_cols - 8)}), ("dout", {0: offset(bf(128, o_cols))}), ("o", {2: f32(128, o_cols)}),
            ("lse", {3: f32(1, heads, 127)}), ("lse", {3: offset(f32(1, heads, 128))}), ("qkv", {1: u8(128, cols)}),
            (mask_name, {4: u8(*mask().shape)}), ("dqkv", {6 + len(kv): bf(128, o_cols)}),
            ("dqkv", {6 + len(kv): f32(128, cols)})])
    if mask_name == "bounds":
        fwd[1].extend([("bounds", {1: i32(1, 128, 3)}), ("bounds", {1: offset(i32(1, 128, 2))}), ("qkv", {1: i32(1, 64, 2)}),
                       ("bounds", {1: i32(0, 128, 2)})])
    else:
        fwd[1].extend([("seq_lens", {1: i32(3)}), ("seq_lens", {1: i32(0)}), ("seq_lens", {1: i32(1, 1)})])
    return fwd, bwd


# binding -> (builder of well-formed CPU arguments, [(argument named by the error, {position: malformed value})])
ROWS = {
    "clip_coef": (lambda: [f32(8), 8, 1.0, 1.0, f32(1), f32(1)],
                  [("partials", {0: f32(4)}), ("partials", {0: u8(32)}), ("partials", {0: strided(f32(8))}),
                   ("coef", {4: f32(0)}), ("norm", {5: i32(1)})]),
    "mse_fwd_bwd": (lambda: [f32(4, 3), f32(4, 3), 1.0],
                    [("out", {0: u8(4, 3)}), ("out", {0: strided(f32(4, 3))}), ("target", {1: f32(4, 2)}),
                     ("target", {1: bf(4, 3)}), ("target", {1: strided(f32(4, 3))})]),
    "xent_fwd_bwd": (lambda: [f32(4, 10), i64(4), -100, 1.0],
                     [("logits", {0: u8(4, 10)}), ("logits", {0: f32(40)}), ("logits", {0: strided(f32(4, 10))}),
                      ("targets", {1: i32(4)}), ("targets", {1: i64(3)})]),
    "lm_loss_fwd": (lambda: [bf(4, 16), bf(8, 16), i64(4), bf(8), -100, None, None, i32(1)],
                    [("hidden", {0: u8(4, 16)}), ("hidden", {0: bf(4, 12)}), ("hidden", {0: bf(0, 16)}), ("weight", {1: bf(8, 8)}),
                     ("weight", {1: bf(6, 16)}), ("weight", {1: strided(bf(8, 16))}), ("targets", {2: i64(3)}), ("bias", {3: bf(7)}),
                     ("rows", {7: i64(1)}), ("lse_out", {5: f32(5)}), ("lse_out", {5: bf(4)}), ("row_loss_out", {6: f32(4)})]),
    "lm_loss_bwd": (lambda: [bf(4, 16), bf(8, 16), i64(4), bf(8), f32(4), f32(5), f32(1), -100, 128, True, True, None, None, None, True],
                    [("hidden", {0: u8(4, 16)}), ("bias", {3: None}), ("lse", {4: f32(3)}), ("row_loss", {5: f32(4)}),
                     ("gscale", {6: f32(2)}), ("gscale", {6: bf(1)}), ("dh_out", {11: bf(4, 8)}), ("dweight_out", {12: f32(8, 16)}),
                     ("rows", {13: i32(2)})]),
    "compact_rows": (lambda: [i64(6), -100, 10],
                     [("targets", {0: i32(6)}), ("targets", {0: i64(0)}), ("targets", {0: i64(2, 3)}), ("targets", {0: strided(i64(6))})]),
    "gather_rows": (lambda: [bf(4, 16), i32(4), i32(1)],
                    [("x", {0: bf(4, 12)}), ("x", {0: u8(4, 16)}), ("index", {1: i32(3)}), ("index", {1: i64(4)}), ("count", {2: i32(2)})]),
    "scatter_rows": (lambda: [bf(4, 16), i32(4), i32(1)],
                     [("dy", {0: bf(4, 12)}), ("dy", {0: f32(4, 16)}), ("index", {1: i32(5)}), ("count", {2: i64(1)})]),
    "gelu_fwd": (lambda: [f32(8), False], [("pre", {0: u8(8)}), ("pre", {0: strided(f32(8))})]),
    "gelu_bwd": (lambda: [f32(8), f32(8), False],
                 [("pre", {1: u8(8)}), ("dy", {0: bf(8)}), ("dy", {0: f32(7)}), ("dy", {0: strided(f32(8))})]),
    "layernorm_fwd": (lambda: [f32(4, 8), f32(8), f32(8), 1e-5],
                      [("x", {0: u8(4, 8)}), ("x", {0: f32(())}), ("gamma", {1: f32(7)}), ("gamma", {1: bf(8)}), ("beta", {2: f32(9)}),
                       ("beta", {2: strided(f32(8))})]),
    "layernorm_bwd": (lambda: [f32(4, 8), f32(4, 8), f32(8), f32(4), f32(4)],
                      [("x", {1: u8(4, 8)}), ("dy", {0: f32(4, 7)}), ("dy", {0: bf(4, 8)}), ("gamma", {2: f32(7)}), ("mean", {3: f32(3)}),
                       ("rstd", {4: bf(4)})]),
    "small_linear_fwd": (lambda: [f32(4, 8), f32(3, 8), f32(3), False],
                         [("x", {0: bf(4, 8)}), ("w", {1: f32(3, 7)}), ("w", {1: strided(f32(3, 8))}), ("b", {2: f32(2)})]),
    "small_linear_bwd": (lambda: [f32(4, 3), f32(4, 8), f32(3, 8), f32(4, 3), False, True, True],
                         [("x", {1: bf(4, 8)}), ("w", {2: f32(3, 7)}), ("y", {3: f32(4, 2)}), ("dy", {0: f32(4, 2)}), ("dy", {0: u8(4, 3)})]),
    "gemm_nt": (lambda: [bf(4, 16), bf(8, 16), bf(8), 0, None],
                [("a", {0: f32(4, 16)}), ("b", {1: bf(8, 8)}), ("bias", {2: bf(7)}), ("bias", {2: strided(bf(8))}),
                 ("out", {4: bf(4, 7)}), ("out", {4: u8(4, 8)}), ("out", {4: strided(bf(4, 8))})]),
    "gemm": (lambda: [bf(4, 16), bf(8, 16), None, False, False, 0, False, None],
             [("a", {0: bf(16)}), ("b", {1: bf(8, 8)}), ("bias", {2: bf(7)}), ("out", {7: i32(4, 8)}), ("out", {7: bf(4, 7)}), ("out", {7: strided(f32(4, 8))})]),
    "gemm_stats": (lambda: [bf(4, 16), bf(8, 16)], [("a", {0: u8(4, 16)}), ("b", {1: bf(8, 8)})]),
    "fp8_amax": (lambda: [bf(16)], [("t", {0: f32(16)}), ("t", {0: strided(bf(16))})]),
    "fp8_cast_transpose": (lambda: [bf(4, 16), f32(1), "e4m3", False, False],
                           [("t", {0: f32(4, 16)}), ("t", {0: bf(())}), ("amax", {1: f32(2)}), ("amax", {1: bf(1)})]),
    "fp8_quantize": (lambda: [bf(4, 16), "e4m3", False, False], [("t", {0: u8(4, 16)}), ("t", {0: strided(bf(4, 16))})]),
    "gemm_fp8": (lambda: [e4m3(4, 16), e4m3(8, 16), f32(1), f32(1), None, 0],
                 [("a", {0: bf(4, 16)}), ("a", {0: offset(e4m3(4, 16))}), ("b", {1: torch.zeros(8, 16, dtype=torch.float8_e5m2)}),
                  ("b", {1: e4m3(8, 32)}), ("a_scale_inv", {2: f32(2)}), ("b_scale_inv", {3: bf(1)}), ("bias", {4: bf(7)})]),
    "rotary": (lambda: [bf(4, 192), i32(4), f32(16, 2, 32), 1, 1, False, 1.0],
               [("x", {0: bf(4, 128)}), ("x", {0: f32(4, 192)}), ("position_ids", {1: i32(3)}), ("position_ids", {1: i64(4)}),
                ("cos_sin", {2: f32(16, 2, 16)}), ("cos_sin", {2: f32(16, 3, 32)})]),
    "qk_norm_rotary_fwd": (lambda: [bf(4, 384), bf(128), bf(128), i32(4), f32(16, 2, 64), 1, 1, 1e-6],
                           [("x", {0: bf(4, 256)}), ("q_weight", {1: bf(64)}), ("k_weight", {2: f32(128)}), ("position_ids", {3: i32(5)}),
                            ("cos_sin", {4: f32(16, 2, 32)})]),
    "qk_norm_rotary_bwd": (lambda: [bf(4, 384), bf(4, 384), f32(4, 2), bf(128), bf(128), i32(4), f32(16, 2, 64), 1, 1],
                           [("dy", {0: bf(4, 256)}), ("x", {1: u8(4, 384)}), ("rstd", {2: f32(7)}), ("rstd", {2: bf(4, 2)}),
                            ("q_weight", {3: bf(129)})]),
    "rmsnorm_fwd": (lambda: [f32(4, 8), f32(8), 1e-6], [("x", {0: u8(4, 8)}), ("gamma", {1: f32(7)}), ("gamma", {1: bf(8)})]),
    "rmsnorm_bwd": (lambda: [f32(4, 8), f32(4, 8), f32(8), f32(4)],
                    [("x", {1: u8(4, 8)}), ("dy", {0: f32(4, 7)}), ("gamma", {2: f32(7)}), ("gamma", {2: bf(8)}), ("rstd", {3: f32(3)})]),
    "swiglu_fwd": (lambda: [bf(4, 32)], [("gate_up", {0: bf(4, 24)}), ("gate_up", {0: f32(4, 32)}), ("gate_up", {0: strided(bf(4, 32))})]),
    "swiglu_bwd": (lambda: [bf(4, 16), bf(4, 32)],
                   [("gate_up", {1: f32(4, 32)}), ("dy", {0: bf(4, 8)}), ("dy", {0: bf(2, 16)}), ("dy", {0: strided(bf(4, 16))})]),
    "geglu_fwd": (lambda: [bf(4, 32)], [("input_gate", {0: bf(4, 40)}), ("input_gate", {0: u8(4, 32)})]),
    "geglu_bwd": (lambda: [bf(4, 16), bf(4, 32)], [("input_gate", {1: bf(4, 24)}), ("dy", {0: bf(4, 32)}), ("dy", {0: f32(4, 16)})]),
    "moe_route": (lambda: [bf(4, 8), 2, False], [("logits", {0: f32(4, 8)}), ("logits", {0: bf(32)})]),
    "moe_router_bwd": (lambda: [bf(4, 8), i32(4, 2), f32(4, 2), f32(8)],
                       [("logits", {0: bf(4, 8, 1)}), ("ids", {1: i32(3, 2)}), ("ids", {1: i64(4, 2)}), ("dgates", {2: f32(4, 3)}),
                        ("dprobsum", {3: f32(7)})]),
    "moe_permute": (lambda: [i32(4, 2), 8], [("ids", {0: i64(4, 2)}), ("ids", {0: i32(8)}), ("ids", {0: strided(i32(4, 2))})]),
    "moe_gather": (lambda: [bf(4, 64), i32(256), 2], [("x", {0: f32(4, 64)}), ("fwd_map", {1: i64(256)}), ("fwd_map", {1: i32(2, 128)})]),
    "moe_gemm": (lambda: [bf(256, 64), bf(2, 32, 64), i32(2), False, None],
                 [("w", {1: bf(2, 32)}), ("a", {0: bf(256, 32)}), ("tile_expert", {2: i32(3)}), ("out", {4: bf(256, 64)}),
                  ("out", {4: f32(256, 32)})]),
    "moe_gemm_wgrad": (lambda: [bf(256, 16), bf(256, 32), i32(3), None],
                       [("a", {0: f32(256, 16)}), ("b", {1: bf(128, 32)}), ("offsets", {2: i64(3)}), ("out", {3: bf(2, 16, 16)})]),
    "moe_combine": (lambda: [bf(256, 64), i32(4, 2), bf(4, 2)],
                    [("y_perm", {0: f32(256, 64)}), ("inv_map", {1: i64(4, 2)}), ("gates", {2: bf(4, 3)})]),
    "moe_combine_bwd": (lambda: [bf(4, 64), bf(256, 64), i32(256), bf(4, 2)],
                        [("dout", {0: bf(4, 64, 1)}), ("y_perm", {1: bf(256, 32)}), ("fwd_map", {2: i32(255)}), ("gates", {3: bf(3, 2)}),
                         ("gates", {3: f32(4, 2)})]),
    "conv_fprop": (lambda: [cl(bf(1, 64, 8, 8)), cl(bf(64, 64, 3, 3)), 1, 1, -1, 0, 0, False, None, 0],
                   [("x", {0: bf(1, 64, 8, 8)}), ("x", {0: cl(f32(1, 64, 8, 8))}), ("w", {1: cl(bf(64, 32, 3, 3))}),
                    ("debug", {8: i64(8)})]),
    "conv_dgrad": (lambda: [cl(bf(1, 64, 8, 8)), cl(bf(64, 32, 3, 3)), 1, 1, -1, 0, 0, 0, None, None, None, None],
                   [("dy", {0: bf(1, 64, 8, 8)}), ("w", {1: cl(bf(32, 32, 3, 3))}), ("addend", {8: cl(bf(1, 32, 8, 4))}),
                    ("bn_x", {9: cl(bf(1, 64, 8, 8)), 11: f32(2, 32)}), ("bn_stats", {9: cl(bf(1, 32, 8, 8))}),
                    ("bn_stats", {9: cl(bf(1, 32, 8, 8)), 11: f32(1, 32)}), ("bn_mask", {10: u8(5)})]),
    "conv_wgrad": (lambda: [cl(bf(1, 64, 8, 8)), cl(bf(1, 32, 8, 8)), 3, 1, 1, 0, 0, 0],
                   [("dy", {0: bf(1, 64, 8, 8)}), ("x", {1: cl(bf(1, 32, 8, 4))}), ("x", {1: cl(f32(1, 32, 8, 8))})]),
    "stem_pack_input": (lambda: [cl(bf(1, 3, 8, 32))], [("x", {0: cl(bf(1, 4, 8, 32))}), ("x", {0: cl(f32(1, 3, 8, 32))})]),
    "stem_pack_weight": (lambda: [cl(bf(64, 3, 7, 7))], [("w", {0: cl(bf(32, 3, 7, 7))}), ("w", {0: bf(64, 3, 7, 7)})]),
    "stem_conv_fprop_packed": (lambda: [bf(1, 7, 40, 8), bf(64, 256), 8, 32, False, True, False],
                               [("xp", {0: bf(1, 7, 32, 8)}), ("xp", {0: f32(1, 7, 40, 8)}), ("w2", {1: bf(64, 128)})]),
    "stem_conv_fprop": (lambda: [cl(bf(1, 3, 8, 32)), cl(bf(64, 3, 7, 7)), False, True],
                        [("x", {0: bf(2, 3, 8, 32)}), ("w", {1: cl(bf(64, 3, 5, 5))})]),
    "stem_conv_wgrad": (lambda: [cl(bf(1, 64, 4, 16)), bf(1, 7, 40, 8), 8, 32, 0, True],
                        [("dy", {0: cl(bf(1, 64, 4, 8))}), ("xp", {1: bf(2, 7, 40, 8)}), ("xp", {1: strided(bf(1, 7, 40, 8))})]),
    "bn_forward": (lambda: [cl(f32(2, 8, 4, 4)), None, f32(8), f32(8), f32(8), f32(8), i64(()), 1e-5, 0.1, True, f32(64), i32(8)],
                   [("x", {0: f32(2, 8, 4, 4)}), ("x", {0: cl(u8(2, 8, 4, 4))}), ("residual", {1: cl(f32(2, 8, 4, 2))}),
                    ("gamma", {2: f32(7)}), ("beta", {3: bf(8)}), ("running_mean", {4: f32(9)}), ("running_var", {5: f32(4)}),
                    ("num_batches", {6: i32(())}), ("partial", {10: i32(64)}), ("counters", {11: f32(8)})]),
    "bn_forward_partials": (lambda: [cl(bf(2, 8, 4, 4)), None, f32(8), f32(8), None, None, None, 1e-5, 0.1, True, f32(2, 3, 8)],
                            [("x", {0: bf(2, 8, 4, 4)}), ("residual", {1: cl(f32(2, 8, 4, 4))}), ("gamma", {2: f32(16)}),
                             ("partial", {10: f32(2, 3, 7)}), ("partial", {10: f32(3, 3, 8)})]),
    "bn_backward_partials": (lambda: [cl(bf(2, 8, 4, 4)), cl(bf(2, 8, 4, 4)), u8(32, 1), f32(8), f32(4, 8), True, False, f32(2, 3, 8)],
                             [("dy", {0: bf(2, 8, 4, 4)}), ("x", {1: cl(u8(2, 8, 4, 4))}), ("y", {2: None}), ("y", {2: u8(32, 2)}),
                              ("gamma", {3: f32(7)}), ("stats", {4: f32(15)}), ("partial", {7: f32(2, 3, 4)})]),
    "bn_backward": (lambda: [cl(f32(2, 8, 4, 4)), cl(f32(2, 8, 4, 4)), u8(32, 1), f32(8), f32(4, 8), True, True, f32(64), i32(8)],
                    [("x", {1: f32(2, 8, 4, 4)}), ("dy", {0: cl(f32(2, 8, 4, 2))}), ("dy", {0: cl(bf(2, 8, 4, 4))}), ("y", {2: None}),
                     ("y", {2: u8(16, 1)}), ("y", {2: i32(32, 1)}), ("gamma", {3: f32(4)}), ("stats", {4: f32(10)}),
                     ("partial", {7: bf(64)}), ("counters", {8: i64(8)})]),
    "maxpool3x3s2_fwd": (lambda: [cl(f32(1, 8, 8, 8))], [("x", {0: cl(u8(1, 8, 8, 8))}), ("x", {0: f32(1, 8, 8, 8)})]),
    "maxpool3x3s2_bwd": (lambda: [cl(f32(1, 8, 4, 4)), cl(u8(1, 8, 4, 4)), 8, 8],
                         [("dy", {0: cl(f32(1, 8, 5, 4))}), ("dy", {0: cl(u8(1, 8, 4, 4))}), ("idx", {1: cl(f32(1, 8, 4, 4))}),
                          ("idx", {1: cl(u8(1, 8, 4, 3))}), ("idx", {1: u8(1, 8, 4, 4)})]),
    "normalize_to_channels_last": (lambda: [f32(2, 3, 4, 4), cl(bf(2, 3, 4, 4)), f32(3), f32(3), 1.0],
                                   [("src", {0: bf(2, 3, 4, 4)}), ("src", {0: strided(f32(2, 3, 4, 4))}), ("dst", {1: bf(2, 3, 4, 4)}),
                                    ("dst", {1: cl(bf(2, 2, 4, 4))}), ("dst", {1: cl(bf(2, 3, 4, 5))}), ("mean", {2: f32(2)}),
                                    ("inv_std", {3: bf(3)})]),
}
for _name, _mask, _mask_name, _heads, _kv, _cols, _hd in (
        ("attention", lambda: i32(1), "seq_lens", 1, None, 192, 64), ("packed_attention", BOUNDS, "bounds", 1, None, 192, 64),
        ("causal_attention", BOUNDS, "bounds", 1, None, 192, 64), ("causal_gqa_attention", BOUNDS, "bounds", 2, 1, 256, 64),
        ("causal_attention_d128", BOUNDS, "bounds", 1, 1, 384, 128)):
    ROWS[_name + "_fwd"], ROWS[_name + "_bwd"] = attn_rows(_mask, _mask_name, _heads, _kv, _cols, _hd)


def _C():
    return _ext.get()


def _takes_tensor(doc):
    """Whether the first line of a pybind docstring (the signature) has a torch.Tensor parameter."""
    params = doc.splitlines()[0].split("->")[0] if doc else ""
    return "torch.Tensor" in params


def test_every_tensor_binding_has_a_row():
    C = _C()
    bindings = {k for k in dir(C) if callable(getattr(C, k)) and not isinstance(getattr(C, k), type) and _takes_tensor(getattr(C, k).__doc__)}
    assert bindings - set(ROWS) - EXEMPT == set(), "bindings without a contract row"
    assert set(ROWS) - bindings == set() and EXEMPT <= bindings


@pytest.mark.parametrize("name", sorted(ROWS))
def test_well_formed_call_reaches_the_device_check(name):
    build, _ = ROWS[name]
    with pytest.raises(RuntimeError, match=rf"^{name}: \w+ must be a CUDA tensor, got cpu"):
        getattr(_C(), name)(*build())


@pytest.mark.parametrize("name,arg,change", [(n, a, c) for n in sorted(ROWS) for a, c in ROWS[n][1]],
                         ids=lambda v: v if isinstance(v, str) else "")
def test_malformed_argument_is_rejected(name, arg, change):
    args = ROWS[name][0]()
    for pos, value in change.items():
        args[pos] = value
    with pytest.raises(RuntimeError, match=rf"^{re.escape(name)}: {arg} must be ") as info:
        getattr(_C(), name)(*args)
    assert "CUDA tensor" not in str(info.value)
