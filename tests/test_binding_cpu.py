"""The ctypes binding without a GPU: the prototypes read from the header, and the operand check every lowlevel wrapper
makes before it calls the library (a missing required tensor is refused on the host, naming the operand)."""
import ctypes
import inspect

import pytest
import torch

from internvideo_b200 import _lib
from internvideo_b200 import lowlevel as ll

# With a GPU, a wrapper that let a None through would hand NULL to a kernel: these cases run only without one.
pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only check")

bf16, f32, i32 = torch.bfloat16, torch.float32, torch.int32


def test_header_parser_maps_each_c_type():
    protos = _lib.parse_prototypes("""
        #define IVB_X 1   /* a comment that names int ivb_not_a_function(int x); */
        const char* ivb_text(void);
        // void ivb_commented_out(void);
        long ivb_sizes(int a, long b, float c, const void* d, float* e,
                       const long long* f, void* stream);
        void ivb_reset(void);
    """)
    vp = ctypes.c_void_p
    assert protos == {
        "ivb_text": (ctypes.c_char_p, []),
        "ivb_sizes": (ctypes.c_long, [ctypes.c_int, ctypes.c_long, ctypes.c_float, vp, vp, vp, vp]),
        "ivb_reset": (None, []),
    }


@pytest.mark.parametrize("decl", ["int ivb_f(double x);", "int ivb_f(unsigned n);", "size_t ivb_f(void);",
                                  "int ivb_f(long long n);"])
def test_header_parser_refuses_unknown_types(decl):
    with pytest.raises(ValueError, match="unknown C type"):
        _lib.parse_prototypes(decl)


def _t(*shape, dtype=bf16):
    return torch.zeros(*shape, dtype=dtype)


# wrapper -> (a complete argument set of CPU tensors, the tensor operands that may not be None)
CASES = {
    "gemm": (dict(a=_t(8, 8), b=_t(8, 8)), ["a", "b"]),
    "gemm_fp8": (dict(a=_t(8, 16, dtype=torch.float8_e4m3fn), a_scale_inv=_t(1, dtype=f32),
                      b=_t(8, 16, dtype=torch.float8_e4m3fn), b_scale_inv=_t(1, dtype=f32)),
                 ["a", "a_scale_inv", "b", "b_scale_inv"]),
    "fp8_quantize": (dict(x=_t(8, 8)), ["x"]),
    "fp8_quantize_rows": (dict(x=_t(8, 8)), ["x"]),
    "norm_fwd_fp8": (dict(x=_t(8, 8, dtype=f32), weight=_t(8)), ["x", "weight"]),
    "norm_fwd": (dict(x=_t(8, 8, dtype=f32), weight=_t(8)), ["x", "weight"]),
    "rmsnorm_pair_fwd": (dict(qkv=_t(8, 24), D=8, w0=_t(8), w1=_t(8), out=_t(8, 24)), ["qkv", "w0", "w1", "out"]),
    "rmsnorm_pair_bwd": (dict(dqk=_t(8, 24), qkv=_t(8, 24), D=8, w0=_t(8), w1=_t(8), rstd=_t(8, 2, dtype=f32)),
                         ["dqk", "qkv", "w0", "w1", "rstd"]),
    "norm_bwd": (dict(dy=_t(8, 8), x=_t(8, 8, dtype=f32), weight=_t(8), mean=None, rstd=_t(8, dtype=f32)),
                 ["dy", "x", "weight", "rstd"]),
    "rmsnorm_bwd_layerscale": (dict(dy=_t(8, 8), x=_t(8, 8, dtype=f32), weight=_t(8), rstd=_t(8, dtype=f32), dx_in=None,
                                    ybr=_t(8, 8), gamma=_t(8), dweight=None, dgamma=None, dcolsum=None),
                               ["dy", "x", "weight", "rstd", "ybr", "gamma"]),
    "layerscale_bwd": (dict(dx=_t(8, 8, dtype=f32), y=None, gamma=None), ["dx"]),
    "colsum": (dict(x=_t(8, 8)), ["x"]),
    "attn_fwd": (dict(q=_t(8, 16), k=_t(8, 16), v=_t(8, 16), B=1, n=8, H=1, d=16, scale=0.25), ["q", "k", "v"]),
    "headaxis_attn_fwd": (dict(qkv=_t(8, 48), B=1, N=8, H=1, d=16, scale=0.25), ["qkv"]),
    "attn_bwd": (dict(q=_t(8, 16), k=_t(8, 16), v=_t(8, 16), out=_t(8, 16), dout=_t(8, 16), lse=_t(1, 1, 8, dtype=f32),
                      B=1, n=8, H=1, d=16, scale=0.25, dq=_t(8, 16), dk=_t(8, 16), dv=_t(8, 16)),
                 ["q", "k", "v", "out", "dout", "lse", "dq", "dk", "dv"]),
    "visible_indices": (dict(mask=_t(1, 8, dtype=torch.bool), n_keep=4), ["mask"]),
    "im2col_visible": (dict(video=_t(1, 3, 2, 16, 16), idx=_t(1, 5, dtype=i32), j0=1, rows_per_clip=4, tubelet=2,
                            patch=8, kpad=384), ["video", "idx"]),
    "gather_add": (dict(src=None, src_bstride=0, table=None, idx=None, idx_bstride=0, idx_off=0, B=1, rows=8, D=8,
                        out=_t(8, 8, dtype=f32), out_bstride=64), ["out"]),
    "scatter_add": (dict(g=_t(8, 8, dtype=f32), g_bstride=64, idx=None, idx_bstride=0, idx_off=0, B=1, rows=8, D=8,
                         table_grad=_t(8, 8, dtype=f32)), ["g", "table_grad"]),
    "ln_l2_fwd": (dict(z=_t(8, 8), weight=_t(8), bias=_t(8)), ["z", "weight", "bias"]),
    "ln_l2_bwd": (dict(z=_t(8, 8), weight=_t(8), bias=_t(8), stats=_t(8, 3, dtype=f32), dout=_t(8, 8)),
                  ["z", "weight", "bias", "stats", "dout"]),
    "vtc_loss_fwd": (dict(cosm=_t(4, 4, dtype=f32), idx=_t(4, dtype=torch.int64), temp=0.07), ["cosm", "idx"]),
    "vtc_loss_bwd": (dict(cosm=_t(4, 4, dtype=f32), idx=_t(4, dtype=torch.int64), temp=0.07, lse_r=_t(4, dtype=f32),
                          lse_c=_t(4, dtype=f32)), ["cosm", "idx", "lse_r", "lse_c"]),
    "l2norm_rows_fwd": (dict(x=_t(8, 8)), ["x"]),
    "l2norm_rows_bwd": (dict(dy=_t(8, 8, dtype=f32), xn=_t(8, 8), inv=_t(8, dtype=f32)), ["dy", "xn", "inv"]),
    "pixel_targets": (dict(video=_t(1, 3, 2, 16, 16), masked_idx=_t(4, dtype=i32), n_mask=4, tubelet=2, patch=8,
                           normalize=True, mean3=_t(3, dtype=f32), std3=_t(3, dtype=f32)),
                      ["video", "masked_idx", "mean3", "std3"]),
    "mse_loss": (dict(pred=_t(8), label=_t(8, dtype=f32), loss_sum=_t(1, dtype=f32)), ["pred", "label"]),
    "adamw_step": (dict(master=_t(8, dtype=f32), exp_avg=_t(8, dtype=f32), exp_avg_sq=_t(8, dtype=f32),
                        grad=_t(8, dtype=f32), param_bf16=_t(8), lr=1e-3, beta1=0.9, beta2=0.95, eps=1e-8, wd=0.05,
                        step=1), ["master", "exp_avg", "exp_avg_sq", "grad", "param_bf16"]),
    "pool_attn_fwd": (dict(q=_t(1, 16), k=_t(8, 16), v=_t(8, 16), B=1, n=8, H=1, d=16, scale=0.25), ["q", "k", "v"]),
    "pool_attn_bwd": (dict(q=_t(1, 16), k=_t(8, 16), v=_t(8, 16), probs=_t(1, 1, 8, dtype=f32), dout=_t(1, 16), B=1,
                           n=8, H=1, d=16, scale=0.25), ["q", "k", "v", "probs", "dout"]),
}


def test_every_wrapper_is_covered():
    wrappers = {name for name, fn in vars(ll).items()
                if inspect.isfunction(fn) and fn.__module__ == ll.__name__ and not name.startswith("_")}
    assert wrappers - {"launch_count", "reset_launch_count", "set_default_2cta", "device_check"} == set(CASES)


@pytest.mark.parametrize("wrapper", sorted(CASES))
def test_missing_required_operand_is_refused_on_the_host(wrapper, monkeypatch):
    monkeypatch.setattr(ll, "_call", lambda *a, **k: pytest.fail(f"{wrapper} reached the library"))
    kwargs, required = CASES[wrapper]
    fn = getattr(ll, wrapper)
    with pytest.raises(_lib.IvbError, match="expected a CUDA tensor"):    # the complete set: refused for the device
        fn(**kwargs)
    for name in required:
        with pytest.raises(_lib.IvbError) as e:
            fn(**{**kwargs, name: None})
        assert str(e.value) == f"{name}: required operand is None"
