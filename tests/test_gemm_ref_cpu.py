"""The float64 GEMM reference and the per-element error metric of tests/gemm_ref.py, checked on the CPU: the GELU forms
against torch and autograd, the RESID / GELU_BWD epilogues against a direct float64 composition, and the metric
against one-ulp errors that a whole-tensor relative norm dilutes."""
import pytest
import torch

import gemm_ref as G

f64 = torch.float64


def _grid():
    return torch.cat((torch.linspace(-12, 12, 4801, dtype=f64), torch.tensor([0.0, 1e-30, -1e-30], dtype=f64)))


@pytest.mark.parametrize("form,approx", [(G.gelu_erf, "none"), (G.gelu_tanh, "tanh")])
def test_gelu_forms_match_torch_and_autograd(form, approx):
    h = _grid().requires_grad_(True)
    f, d1, d2, e0, e1 = form(h.detach())
    ft = torch.nn.functional.gelu(h, approximate=approx)
    torch.testing.assert_close(f, ft.detach(), rtol=1e-13, atol=1e-15)   # torch cancels in the left tail
    (g1,) = torch.autograd.grad(ft.sum(), h, create_graph=True)
    (g2,) = torch.autograd.grad(g1.sum(), h)
    torch.testing.assert_close(d1, g1.detach(), rtol=1e-12, atol=1e-13)
    torch.testing.assert_close(d2, g2, rtol=1e-10, atol=1e-12)
    assert (e0 >= 0).all() and (e1 > 0).all()


def test_gelu_error_terms():
    """The documented form errors: A-S is absolute on Phi (7.5e-8, times |h| for the value); tanh.approx is about
    2^-11 of t, which for the value is half of it times |h|."""
    h = torch.tensor([-10.0, -5.0, 0.0, 3.0], dtype=f64)
    _, _, _, e0, e1 = G.gelu_erf(h)
    assert abs(float(e0[0]) - 7.5e-7) < 1e-9 and abs(float(e0[1]) - 3.75e-7) < 1e-9
    assert float(e0[2]) == 0.0 and abs(float(e1[2]) - 7.5e-8 - G.EVAL * 0.5) < 1e-12
    _, _, _, t0, _ = G.gelu_tanh(h)
    assert abs(float(t0[3]) / (1.5 * G.TANH_REL * float(torch.tanh(G.TANH_C * (h[3] + G.TANH_A * h[3] ** 3)))) - 1) < 1e-2


def _bf(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16)


@pytest.mark.parametrize("layout", ["nt", "dgrad", "wgrad"])
def test_resid_reference_is_the_direct_composition(layout):
    M, N, K = 37, 48, 24
    a = _bf((K, M) if layout == "wgrad" else (M, K), 1)
    b = _bf((K, N) if layout != "nt" else (N, K), 2, 0.1)
    a_t, b_t = layout == "wgrad", layout != "nt"
    bias, gamma = _bf((N,), 3, 0.1), _bf((N,), 4) * 1e-5
    aux = torch.randn((M, N), generator=torch.Generator().manual_seed(5))
    rs = torch.tensor([0.0, 1.0 / 0.75] * 18 + [1.0])
    am = (a.t() if a_t else a).double()
    bm = (b if b_t else b.t()).double()
    y = am @ bm + bias.double()
    (o0, s0), (o1, s1) = G.gemm_ref(a, b, a_t=a_t, b_t=b_t, epi=G.EPI_RESID, bias=bias, gamma=gamma, aux=aux,
                                    rowscale=rs, out1=torch.empty(1))
    torch.testing.assert_close(o0, aux.double() + rs.double()[:, None] * gamma.double() * y, rtol=1e-15, atol=0)
    torch.testing.assert_close(o1, y, rtol=1e-15, atol=0)
    assert torch.equal(o0[0::2][:18], aux.double()[0::2][:18])           # rowscale 0: the residual itself
    assert (s0[0::2][:18] == 0).all() and (s0[1::2] > 0).all() and (s1 > 0).all()
    (p0, _), = G.gemm_ref(a, b, a_t=a_t, b_t=b_t, epi=G.EPI_RESID, aux=aux)
    torch.testing.assert_close(p0, aux.double() + am @ bm, rtol=1e-15, atol=0)


@pytest.mark.parametrize("flags", [0, G.FLAG_GELU_TANH, G.FLAG_GELU_SAVE_GRAD])
def test_gelu_bwd_reference_is_the_direct_composition(flags):
    M, N, K = 33, 40, 16
    a, b = _bf((M, K), 6), _bf((N, K), 7, 0.1)
    aux = _bf((M, N), 8, 2.0)
    acc = a.double() @ b.double().t()
    hv = aux.double().requires_grad_(True)
    if flags & G.FLAG_GELU_SAVE_GRAD:
        want = acc * aux.double()
    else:
        f = torch.nn.functional.gelu(hv, approximate="tanh" if flags & G.FLAG_GELU_TANH else "none")
        (d,) = torch.autograd.grad(f.sum(), hv)
        want = acc * d
    (o, s), = G.gemm_ref(a, b, epi=G.EPI_GELU_BWD, flags=flags, aux=aux)
    torch.testing.assert_close(o, want, rtol=1e-12, atol=1e-15)
    assert (s > 0).all()


@pytest.mark.parametrize("save", [False, True])
def test_bias_gelu_and_accum_references(save):
    M, N, K = 20, 24, 16
    a, b, bias = _bf((M, K), 9), _bf((N, K), 10, 0.2), _bf((N,), 11)
    h = a.double() @ b.double().t() + bias.double()
    fl = G.FLAG_GELU_TANH | (G.FLAG_GELU_SAVE_GRAD if save else 0)
    (g, _), (o1, _) = G.gemm_ref(a, b, epi=G.EPI_BIAS_GELU, flags=fl, bias=bias, out1=torch.empty(1))
    hv = h.clone().requires_grad_(True)
    f = torch.nn.functional.gelu(hv, approximate="tanh")
    (d,) = torch.autograd.grad(f.sum(), hv)
    torch.testing.assert_close(g, f.detach(), rtol=1e-13, atol=1e-15)
    torch.testing.assert_close(o1, d if save else h, rtol=1e-12, atol=1e-15)
    old = _bf((M, N), 12)
    (acc, _), = G.gemm_ref(a, b, flags=G.FLAG_ACCUM, bias=bias, out0=old)
    torch.testing.assert_close(acc, h + old.double(), rtol=1e-15, atol=0)


# ---------------------------------------------------------------- the metric
M_, N_ = 417, 1000


def _exact_pair():
    """A bf16 result equal to its reference: every error is 0 until one is planted."""
    got = _bf((M_, N_), 20)
    return got, got.double(), torch.zeros((M_, N_), dtype=f64)


def _plant_ulp(got, rows, cols):
    bits = got.view(torch.int16).clone()
    bits[rows, cols] += 1                 # one ulp away from zero (no element here is 0 or at a binade's end)
    return bits.view(torch.bfloat16)


@pytest.mark.parametrize("rows,cols,where", [
    (slice(130, 131), slice(272, 288), "tile (1, 2) of 128x128, warpgroup band 0 (rows 128..191), epilogue chunk 1"),
    (slice(320, 384), slice(0, 1000), "tile (2, "),
    (slice(0, 417), slice(992, 1000), "epilogue chunk 6 (cols 992..1007), last column tile (104 cols)"),
])
def test_metric_flags_a_one_ulp_error_the_global_norm_misses(rows, cols, where):
    got, ref, scale = _exact_pair()
    assert float(G.elem_errors(got, ref, scale).max()) == 0.0
    bad = _plant_ulp(got, rows, cols)
    errs = G.elem_errors(bad, ref, scale)
    e, desc = G.worst(errs)
    assert 1.9 < e <= 2.0, e                                  # one ulp = two half-ulps
    assert where in desc, desc
    flagged = errs > 1.0
    assert flagged[rows, cols].all() and int(flagged.sum()) == flagged[rows, cols].numel()
    glob = float((bad.double() - ref).norm() / ref.norm())
    assert glob < 6e-3, glob                                  # what a relative norm over the whole tensor sees


def test_metric_band_and_ragged_rows():
    got, ref, scale = _exact_pair()
    bad = _plant_ulp(got, slice(400, 417), slice(0, 16))     # rows of the ragged last tile of 128 (and of 256)
    e, desc = G.worst(G.elem_errors(bad, ref, scale), bm=256, bn=176)
    assert "tile (1, 0) of 256x176, warpgroup band 2 (rows 384..447)" in desc and "last row tile (161 rows)" in desc


def test_metric_within_half_ulp_and_nan():
    ref = torch.tensor([1.0 + 2 ** -9, 3.0e-3, -7.0, 0.0, 1e-40], dtype=f64)
    got = ref.to(torch.bfloat16)
    assert float(G.elem_errors(got, ref, torch.zeros_like(ref)).max()) <= 1.0
    got32 = ref.float()
    assert float(G.elem_errors(got32, ref, torch.zeros_like(ref)).max()) <= 1.0
    nan = got.clone()
    nan[2] = float("nan")
    errs = G.elem_errors(nan, ref, torch.zeros_like(ref))
    assert errs[2] == float("inf") and float(errs[[0, 1, 3, 4]].max()) <= 1.0


def test_binned_bias_sees_a_systematic_error_inside_the_tolerance():
    """The erf derivative in place of the tanh one is at most 8.7e-4 off: inside the tanh form's per-element tolerance
    (tanh.approx.f32 is allowed 2^-11 of t), but the same way for every h in a bin, which correct rounding is not."""
    h = (torch.randn(400000, generator=torch.Generator().manual_seed(30), dtype=f64) * 1.5).to(torch.bfloat16).double()
    _, ref, _, _, scale = G.gelu_tanh(h)
    wrong = G.gelu_erf(h)[1].to(torch.bfloat16)
    assert float(G.elem_errors(wrong, ref, scale).max()) < 1.3
    e_ok, _ = G.binned_bias(ref.to(torch.bfloat16), ref, scale, h)
    assert e_ok == 0.0, e_ok
    e_bad, edge = G.binned_bias(wrong, ref, scale, h)
    assert e_bad > 0.5 and -2.0 <= edge <= 1.0, (e_bad, edge)
