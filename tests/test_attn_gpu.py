"""wgmma attention forward/backward, head-axis attention and pool attention against float64 references (gpu).

Token-axis attention runs in four forms, each its own set of kernel instantiations: plain (ivb_attn_fwd /
ivb_attn_bwd), causal (ivb_attn_{fwd,bwd}_causal), key-length (ivb_attn_fwd_keylen, forward only) and DropPath plan
(ivb_attn_{fwd,bwd}_plan).  Causal and key-length results are compared with the masked float64 reference; the plan
form's kept clips must give the plain call's bits and its dropped clips zeros.  Masked keys contribute exactly 0 to P,
so replacing what a mask hides must leave the other rows' bits alone (the exact-masking tests).

Errors are measured per (clip, head, 64-row band) with tests/attn_ref.py:tile_errors, so an error confined to one
item, one warpgroup's rows or the ragged last tile is not diluted by the rest of the tensor.  lse2 is checked in
absolute log2 units.  Every limit is at most twice the worst value measured over this file on an H100 80GB HBM3
(SXM, 400 W power limit) with the kernels as committed; the measured worst is the comment beside each limit.
The worst bands are mostly the ragged last band of a single row, where the rms is taken over one row.  The causal
form keeps these limits except where its own key says otherwise; those were measured on an H100 80GB HBM3 at a 700 W
power limit, where the plain form's worst values came out as listed here.
"""
import ctypes

import pytest
import torch

from attn_ref import attn_ref_bwd, attn_ref_fwd, tile_errors, worst

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
NAN16 = torch.tensor(float("nan"), dtype=bf16).view(torch.int16).item()
NAN32 = torch.tensor(float("nan"), dtype=torch.float32).view(torch.int32).item()

LIMITS = {
    # token-axis attention on N(0, 1)-like inputs: tile error of O / dQ / dK / dV, max |lse2 error| (log2 units)
    "o": 1.2e-2,                 # measured 6.03e-3
    "lse": 1.0e-5,               # 5.39e-6
    "dq": 1.3e-2,                # 6.51e-3
    "dk": 1.3e-2,                # 6.54e-3
    "dv": 9.5e-3,                # 4.97e-3
    # causal dV: key j is attended by the n - j queries >= j, so the first keys' dV rows are several times the head's
    # rms (about sqrt(n / 64) at n = 2049) and a band of them errs by more relative to it
    "dv_causal": 2.0e-2,         # 1.03e-2 (n = 2049, rows 0..63)
    # n = 2: each row of dS is two terms that cancel
    "dq_two_keys": 2.7e-2,       # 1.39e-2
    "dk_two_keys": 2.6e-2,       # 1.35e-2
    # gradients that vanish in exact arithmetic (n = 1; dQ with identical keys): max |value|, inputs of unit scale
    "dq_vanishing": 2.7e-3,      # 1.37e-3
    "dk_vanishing": 4.8e-7,      # 2.44e-7
    # score distributions
    "o_peaked": 3.3e-3,          # 1.67e-3
    "lse_peaked": 4.4e-5,        # 2.23e-5
    "dq_peaked": 1.4e-2,         # 7.38e-3
    "dk_peaked": 1.5e-2,         # 7.89e-3
    "dv_peaked": 4.9e-3,         # 2.45e-3
    "o_offset": 4.0e-3,          # 2.00e-3
    "lse_offset": 4.4e-4,        # 2.23e-4 (|lse2| ~ 1000)
    "dk_offset": 1.25e-2,        # 6.34e-3
    "dv_offset": 1.1e-2,         # 5.56e-3
    "o_uniform": 3.7e-3,         # 1.86e-3
    "lse_uniform": 3.6e-6,       # 1.84e-6
    "dk_uniform": 4.8e-3,        # 2.44e-3
    "dv_uniform": 6.6e-3,        # 3.34e-3
    # causal, identical keys: a row with few keys has an O of the size of V's rows, so the bf16 rounding of O in
    # delta = rowsum(dO * O) no longer cancels in dS's row sum; and the first keys' dK rows are skewed as dV's above
    "dq_vanishing_causal": 2.4e-2,   # 1.22e-2 (d = 88)
    "dk_uniform_causal": 1.1e-2,     # 5.74e-3
    "o_rescale": 3.5e-3,         # 1.76e-3
    "lse_rescale": 5.6e-5,       # 2.85e-5
    "dq_rescale": 3.6e-2,        # 1.81e-2
    "dk_rescale": 2.2e-2,        # 1.12e-2
    "dv_rescale": 1.2e-2,        # 6.06e-3
    # head-axis attention: tile error of O
    "headaxis": 3.8e-3,          # 1.90e-3
    # pool attention: per-(clip, head) error of out / dq, tile error of dk / dv, max |error| of probs and row sums
    "pool_o": 3.9e-3,            # 1.96e-3
    "pool_probs": 8.0e-8,        # 4.08e-8
    "pool_probs_sum": 3.5e-7,    # 1.78e-7
    "pool_dq": 4.0e-3,           # 2.03e-3
    "pool_dk": 1.45e-2,          # 7.48e-3
    "pool_dv": 2.5e-2,           # 1.27e-2
}


def _within(kind, value, where=None):
    assert value <= LIMITS[kind], f"{kind}: {value:.3e} > {LIMITS[kind]:.1e} at {where}"


def _tiles(kind, got, ref, B, n, H, d):
    """Largest per-(clip, head, 64-row band) error of a [B*n, H*d] result; the failure names the (b, h, band)."""
    e, (b, h, band) = worst(tile_errors(got, ref, B, n, H, d))
    _within(kind, e, f"clip {b}, head {h}, rows {64 * band}..{min(n, 64 * band + 64) - 1}")


def _lse(kind, got, ref):
    e, (b, h, q) = worst((got.double() - ref).abs())
    _within(kind, e, f"clip {b}, head {h}, query {q}")


def _ll():
    from internvideo_b200 import lowlevel
    return lowlevel


def _randn(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g) * scale


# Every head dim the ABI accepts, and the kernel instantiation (KA, NO, KS) it selects in the forward and in both
# passes of the backward: KA = 64-wide atoms covering d, NO = d rounded up to 32 (the wgmma N of O += P V and of the
# gradient MMAs), KS = ceil(d / 16) k16 steps of S = Q K^T, which is NO/16 or NO/16 - 1.
#   d   16: (1, 32, 1)   24, 32: (1, 32, 2)    40, 48: (1, 64, 3)    56, 64: (1, 64, 4)
#   d 72, 80: (2, 96, 5)   88, 96: (2, 96, 6)   104, 112: (2, 128, 7)  120, 128: (2, 128, 8)
HEAD_DIMS = list(range(16, 129, 8))
# n = 190: the last 128-row block has one live warpgroup (62 rows) and a ragged 62-key tile.
# n = 353 with 24 heads and 2 clips: 144 CTAs (more than one wave on 132 SMs); the last block has two live
# warpgroups (97 rows).
DIM_CASES = [(2, 190, 3, d) for d in HEAD_DIMS] + [(2, 353, 24, d) for d in HEAD_DIMS]
# Sequence boundaries around the 64-key tile and the 128-row block, including n mod 128 = 64 past one block, where
# the last block's live warpgroups go from 2 to 1.
SEQ_CASES = [(2, n, 3, d) for d in (64, 88)
             for n in (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 385)]
# The shapes the project runs: InternVideo2 1B (d = 88), 6B (25 heads of 128) and a 2049-token clip.
MODEL_CASES = [(2, 417, 16, 88), (1, 833, 25, 128), (1, 2049, 16, 64)]
# Grids larger than one wave, 1, 2, 4 and 9 key tiles per block, single-item grids.
MISC_CASES = [(1, 64, 2, 64), (2, 209, 6, 64), (1, 1025, 4, 64), (1, 833, 5, 128), (3, 13, 2, 64), (1, 128, 1, 88),
              (1, 1568, 2, 88), (1, 129, 3, 128), (5, 417, 16, 88), (40, 64, 4, 64), (6, 300, 25, 64),
              (2, 1025, 16, 64), (20, 144, 8, 128), (3, 257, 40, 32), (6, 256, 25, 64), (1, 200, 1, 88),
              (1, 1025, 2, 64), (1, 833, 3, 128)]
# The text towers' shapes: MobileCLIP's causal 77 tokens, one whole block, 200 = a second block with one live warpgroup
# and a ragged key tile, 417 and 1025 (17 key tiles); BERT captions of 40 tokens (one key tile), 77 and 193 tokens.
TEXT_CASES = [(2, 77, 8, 64), (2, 128, 8, 64), (2, 200, 16, 88), (2, 417, 4, 64), (2, 1025, 2, 128), (64, 40, 16, 64),
              (4, 77, 8, 64), (3, 193, 4, 40)]
CASES = DIM_CASES + SEQ_CASES + MODEL_CASES + MISC_CASES + TEXT_CASES
assert len(set(CASES)) == len(CASES)

FORMS = ("plain", "causal", "keylen", "plan")
BWD_FORMS = ("plain", "causal", "plan")          # the key-length form has no backward


def _formed(cases, forms=FORMS):
    """pytest params (*case, form) of every case in every form; the plain form keeps the case's own id."""
    return [pytest.param(*c, f, id="-".join(map(str, c)) + ("" if f == "plain" else f"-{f}"))
            for c in cases for f in forms]


def _key_lengths(B, n, shift):
    """int32 [B]: clip b keeps the ((b + shift) mod m)-th of the m lengths in {1, 63, 64, 65, 127, 128, 129, n - 1, n}
    that lie in [1, n] (either side of the 64-key tile and the 128-row block)."""
    vals = sorted({x for x in (1, 63, 64, 65, 127, 128, 129, n - 1, n) if 1 <= x <= n})
    return torch.tensor([vals[(b + shift) % len(vals)] for b in range(B)], device="cuda", dtype=torch.int32)


def _key_shifts(B, n):
    """Shifts of _key_lengths whose calls together give every length to some clip."""
    return range(0, len({x for x in (1, 63, 64, 65, 127, 128, 129, n - 1, n) if 1 <= x <= n}), B)


def _plan_rows(B, n, draw):
    """fp32 [B*n] DropPath factors keeping clip b when b + draw is even: draws 0 and 1 keep and drop every clip once."""
    keep = (torch.arange(B, device="cuda") + draw) % 2 == 0
    return torch.where(keep, 1.25, 0.0).float().repeat_interleave(n)


def _form_kw(form, B, n, draw=0):
    """attn_fwd's keyword arguments for a form: causal, kv_len (_key_lengths) or rowscale (_plan_rows)."""
    return {"causal": form == "causal", "kv_len": _key_lengths(B, n, draw) if form == "keylen" else None,
            "rowscale": _plan_rows(B, n, draw) if form == "plan" else None}


def _pad_keys(k, v, kv, n, seed):
    """The keys >= kv[b] of each clip's k and v rows set to +-1e4 (in place): a padded key the kernel fails to mask
    dominates its row."""
    big = torch.where(_randn(n, 2 * k.shape[1], seed=seed) > 0, 1e4, -1e4).to(bf16)
    for b, kb in enumerate(kv.tolist()):
        k[b * n + kb:(b + 1) * n] = big[kb:, :k.shape[1]]
        v[b * n + kb:(b + 1) * n] = big[kb:, k.shape[1]:]


def _packed(B, n, H, d, seed, scale=1.0):
    """q, k, v as the three slots of one packed [B*n, 3*H*d] bf16 buffer (the FlashAttention qkv layout)."""
    D = H * d
    qkv = _randn(B * n, 3 * D, scale=scale, seed=seed).to(bf16)
    return qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]


def _grad_slots(B, n, H, d):
    """dq, dk, dv as the slots of one NaN-filled [B*n, 3*H*d] buffer: an element the kernel skips stays NaN."""
    D = H * d
    g = torch.full((B * n, 3 * D), float("nan"), device="cuda", dtype=bf16)
    return g[:, :D], g[:, D:2 * D], g[:, 2 * D:]


def _check_fwd(q, k, v, B, n, H, d, scale, tag="", causal=False, kv_len=None):
    out, lse = _ll().attn_fwd(q, k, v, B, n, H, d, scale, causal=causal, kv_len=kv_len)
    o_ref, lse_ref = attn_ref_fwd(q, k, v, B, n, H, d, scale, causal=causal, kv_len=kv_len)
    _tiles("o" + tag, out, o_ref, B, n, H, d)
    _lse("lse" + tag, lse, lse_ref)
    return out, lse, lse_ref


def _check_bwd(q, k, v, dout, B, n, H, d, scale, tag="", vanishing=(), skip=(), kinds=None, causal=False):
    """The backward once with the forward kernel's lse2 and once with the float64 reference's rounded to fp32, so
    an lse2 error of the forward cannot hide inside the backward's tolerance.  Gradients named in `vanishing` are
    exactly zero in exact arithmetic (the terms of dS K or dS^T Q cancel): their largest magnitude is checked, as a
    relative error would divide by zero.  `kinds` maps a gradient's name to its LIMITS key where that is not
    name + tag (name + "_vanishing" for those).  Returns the first run's gradients."""
    out, lse, lse_ref = _check_fwd(q, k, v, B, n, H, d, scale, tag, causal=causal)
    refs = attn_ref_bwd(q, k, v, dout, B, n, H, d, scale, causal=causal)
    first = None
    for lse_in in (lse, lse_ref.float()):
        grads = _grad_slots(B, n, H, d)
        _ll().attn_bwd(q, k, v, out, dout, lse_in, B, n, H, d, scale, *grads, causal=causal)
        for name, got, ref in zip(("dq", "dk", "dv"), grads, refs):
            if name in vanishing:
                assert bool(torch.isfinite(got).all()), name
                _within((kinds or {}).get(name, name + "_vanishing"), float(got.float().abs().max()))
            elif name not in skip:
                _tiles((kinds or {}).get(name, name + tag), got, ref, B, n, H, d)
        first = first or grads
    return first


def _check_plan(q, k, v, dout, B, n, H, d, scale):
    """The plan form under draws 0 and 1 of _plan_rows against the plain call: a kept clip's out and lse (and, with
    dout, dq, dk and dv) have the plain call's bits; a dropped clip's are all 0."""
    plain = _fwd_bwd(q, k, v, dout, B, n, H, d, scale)
    for draw in (0, 1):
        rs = _plan_rows(B, n, draw)
        kept = rs[::n] != 0
        got = _fwd_bwd(q, k, v, dout, B, n, H, d, scale, rowscale=rs)
        for name, a, ref in zip(("out", "lse", "dq", "dk", "dv"), _flat(got), _flat(plain)):
            a, ref = a.reshape(B, -1), ref.reshape(B, -1)
            assert torch.equal(a[kept], ref[kept]), (draw, name, "kept clips")
            assert int(a[~kept].count_nonzero()) == 0, (draw, name, "dropped clips")


@pytest.mark.parametrize("B,n,H,d,form", _formed(CASES))
def test_attn_fwd(cuda_lib, B, n, H, d, form):
    seed = B * 1000 + n + d
    if form == "plan":
        _check_plan(*_packed(B, n, H, d, seed=seed, scale=1.5), None, B, n, H, d, d ** -0.5)
    elif form == "keylen":
        for shift in _key_shifts(B, n):           # every length in some clip
            kv = _key_lengths(B, n, shift)
            q, k, v = _packed(B, n, H, d, seed=seed + shift, scale=1.5)
            _pad_keys(k, v, kv, n, seed=shift)
            _check_fwd(q, k, v, B, n, H, d, d ** -0.5, kv_len=kv)
    else:
        _check_fwd(*_packed(B, n, H, d, seed=seed, scale=1.5), B, n, H, d, d ** -0.5, causal=form == "causal")


@pytest.mark.parametrize("B,n,H,d,form", _formed(CASES, BWD_FORMS))
def test_attn_bwd(cuda_lib, B, n, H, d, form):
    q, k, v = _packed(B, n, H, d, seed=B * 77 + n + d)
    dout = _randn(B * n, H * d, seed=n + 5).to(bf16)
    if form == "plan":
        _check_plan(q, k, v, dout, B, n, H, d, d ** -0.5)
        return
    # one key: P = 1 and dS = 0, so dQ and dK vanish; two keys: dQ and dK are differences of two close terms (causal:
    # in row 1)
    kinds = {"dq": "dq_two_keys", "dk": "dk_two_keys"} if n == 2 else {}
    if form == "causal":
        kinds["dv"] = "dv_causal"
    _check_bwd(q, k, v, dout, B, n, H, d, d ** -0.5, vanishing=("dq", "dk") if n == 1 else (), kinds=kinds,
               causal=form == "causal")


# ------------------------------------------------------------------------------------------- score distributions
def _score_rows(q, k, B, n, H, d, scale):
    """float64 scaled scores of clip 0, [H, n, n]."""
    qh, kh = (t[:n].double().reshape(n, H, d).transpose(0, 1) for t in (q, k))
    return (qh @ kh.transpose(-2, -1)) * scale


# causal: the same inputs, each row over its keys <= query
SCORE_FORMS = [pytest.param(d, causal, id=f"{d}-causal" if causal else f"{d}")
               for d in (64, 88) for causal in (False, True)]


@pytest.mark.parametrize("d,causal", SCORE_FORMS)
def test_attn_peaked_scores(cuda_lib, d, causal):
    """Scores spread over 30+ nats per row: P is close to one-hot and most exp2 terms underflow."""
    B, n, H = 2, 300, 4
    q, k, v = _packed(B, n, H, d, seed=11)
    q = (q.float() * 12).to(bf16)
    s = _score_rows(q, k, B, n, H, d, d ** -0.5)
    assert float((s.amax(-1) - s.amin(-1)).min()) > 30
    _check_bwd(q, k, v, _randn(B * n, H * d, seed=12).to(bf16), B, n, H, d, d ** -0.5, "_peaked", causal=causal)


@pytest.mark.parametrize("d,causal", SCORE_FORMS)
def test_attn_offset_keys(cuda_lib, d, causal):
    """A large vector c added to every key of a (clip, head), with q leaning towards c: each row's scaled scores sit
    hundreds of units from zero.  Softmax is invariant to the shift, so this tests the running-max subtraction and
    lse2 at large magnitude against the float64 reference on the same rounded inputs."""
    B, n, H = 2, 300, 4
    D = H * d
    u = torch.where(_randn(B, 1, D, seed=21) > 0, 1.0, -1.0)
    q = (_randn(B, n, D, seed=22) + 2 * u).reshape(B * n, D).to(bf16)
    k = (_randn(B, n, D, seed=23) + 40 * u).reshape(B * n, D).to(bf16)
    v = _randn(B * n, D, seed=24).to(bf16)
    s = _score_rows(q, k, B, n, H, d, d ** -0.5)
    assert float(s.mean(-1).abs().min()) > 200
    # dQ = scale * dS K is not checked here: K's common part is 40x the part that differs between keys, so the bf16
    # rounding of dS before its MMA alone gives dQ a ~15 % error (measured 0.17), in any bf16-dS kernel.
    _check_bwd(q, k, v, _randn(B * n, D, seed=25).to(bf16), B, n, H, d, d ** -0.5, "_offset", skip=("dq",),
               causal=causal)


@pytest.mark.parametrize("d,causal", SCORE_FORMS)
def test_attn_identical_keys(cuda_lib, d, causal):
    """Every key of a (clip, head) equal: P is uniform, 1/n (causal: 1/(query + 1)), over a ragged last tile, and
    dQ = scale * dS K vanishes because each row of dS sums to zero."""
    B, n, H = 2, 300, 4
    q, _, v = _packed(B, n, H, d, seed=31)
    k = _randn(B, 1, H * d, seed=32).expand(B, n, H * d).reshape(B * n, H * d).to(bf16)
    _check_bwd(q, k, v, _randn(B * n, H * d, seed=33).to(bf16), B, n, H, d, d ** -0.5, "_uniform",
               vanishing=("dq",), causal=causal,
               kinds={"dq": "dq_vanishing_causal", "dk": "dk_uniform_causal"} if causal else None)


@pytest.mark.parametrize("d,causal", SCORE_FORMS)
def test_attn_zero_dout_rows(cuda_lib, d, causal):
    """Rows of dO that are exactly zero (every 7th query, and the whole band of rows 128..191) have dS = 0, so their
    dQ rows are exactly zero; the other gradients still match the reference."""
    B, n, H = 2, 300, 4
    q, k, v = _packed(B, n, H, d, seed=41)
    dout = _randn(B * n, H * d, seed=42)
    zero = torch.zeros(B * n, dtype=torch.bool, device="cuda")
    zero[::7] = True
    zero[128:192] = True
    dout[zero] = 0
    dq, _, _ = _check_bwd(q, k, v, dout.to(bf16), B, n, H, d, d ** -0.5, causal=causal)
    assert int(dq[zero].count_nonzero()) == 0


def test_attn_fwd_rescale_path(cuda_lib):
    """Scores that grow along the key axis move the running max at every tile: the O rescale by alpha runs in
    every key tile of every row block, plain and causal."""
    B, n, H, d = 1, 300, 2, 64
    D = H * d
    q = _randn(B * n, D, seed=1)
    k = _randn(B * n, D, seed=2)
    ramp = torch.linspace(0, 6, n, device="cuda")[:, None]
    k = k + ramp * q.mean(0, keepdim=True).sign() * 0.5
    q = (q.abs() * q.mean(0, keepdim=True).sign()).to(bf16)
    v = _randn(B * n, D, seed=3).to(bf16)
    for causal in (False, True):
        _check_bwd(q, k.to(bf16), v, _randn(B * n, D, seed=4).to(bf16), B, n, H, d, 0.5, "_rescale", causal=causal)


# ------------------------------------------------------------------------------------------- the model's layouts
class _Buf:
    """A bf16/fp32 operand as a [rows, cols] view at column `col0` of a NaN-filled [rows + spare, pitch] buffer."""

    def __init__(self, rows, cols, pitch, col0=0, spare=0, dtype=bf16):
        self.base = torch.full((rows + spare, pitch), float("nan"), device="cuda", dtype=dtype)
        self.view = self.base[:rows, col0:col0 + cols]
        self.inside = torch.zeros(self.base.shape, dtype=torch.bool, device="cuda")
        self.inside[:rows, col0:col0 + cols] = True

    def fill(self, x):
        self.view.copy_(x)
        return self

    def check_poison(self, name):
        """Every element of the view is finite; every element outside it is still the NaN it was filled with."""
        bits = self.base.view(torch.int16 if self.base.dtype == bf16 else torch.int32)
        assert bool(torch.isfinite(self.base[self.inside]).all()), f"{name}: non-finite element inside the view"
        outside = bits[~self.inside]
        nan = NAN16 if self.base.dtype == bf16 else NAN32
        assert bool((outside == nan).all()), f"{name}: {int((outside != nan).sum())} elements outside the view written"


FWD_ENTRY = {"plain": "ivb_attn_fwd", "causal": "ivb_attn_fwd_causal", "keylen": "ivb_attn_fwd_keylen",
             "plan": "ivb_attn_fwd_plan"}


def _attn_fwd_raw(q, k, v, out, lse, B, n, H, d, scale, form="plain", kv_len=None, rowscale=None, **_):
    """The form's forward entry point through the C ABI with a caller-owned lse2 buffer (the wrapper allocates its
    own)."""
    from internvideo_b200 import _lib
    extra = [x.data_ptr() for x in (kv_len, rowscale) if x is not None]
    rc = getattr(_lib.load(), FWD_ENTRY[form])(
        q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.data_ptr(), out.stride(0),
        lse.data_ptr(), B, n, H, d, ctypes.c_float(scale), *extra, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, FWD_ENTRY[form])


@pytest.mark.parametrize("layout", ["model", "own_pitches"])
@pytest.mark.parametrize("B,n,H,d,form", _formed([(2, 417, 16, 88), (3, 193, 4, 40), (1, 833, 25, 128)]))
def test_attn_model_layout_poisoned(cuda_lib, layout, B, n, H, d, form):
    """Operands laid out as ops.block_forward / block_backward lay them out: q, k in the [M, 2D] q/k-norm buffer,
    v in [M, 3D] qkv, out and dout [M, D], dq/dk/dv the slots of [M, 3D].  "own_pitches" gives every operand its own
    buffer with pad columns beyond the view and spare rows after B*n.  Everything outside the views, inputs and
    outputs, is NaN, and so are the output views before the call: a read outside a view makes a result non-finite,
    a skipped element stays NaN, a write outside a view changes NaN bits.  The key-length form runs the forward only;
    the plan form keeps clips 0, 2, ... and its reference is 0 for the others."""
    M, D = B * n, H * d
    scale = d ** -0.5
    if layout == "model":
        qkn, qkv, a, da, dqkv = (_Buf(M, c, c) for c in (2 * D, 3 * D, D, D, 3 * D))
        qkn.fill(_randn(M, 2 * D, seed=51))
        qkv.view[:, 2 * D:] = _randn(M, D, seed=52).to(bf16)
        qkv.inside[:, :2 * D] = False                     # the pre-norm q, k slots are not attention's to read
        da.fill(_randn(M, D, seed=53))
        q, k, v = qkn.view[:, :D], qkn.view[:, D:], qkv.view[:, 2 * D:]
        dq, dk, dv = dqkv.view[:, :D], dqkv.view[:, D:2 * D], dqkv.view[:, 2 * D:]
        bufs = {"qkv": qkv, "a": a, "dqkv": dqkv}
        out, dout = a.view, da.view
    else:
        spec = {"q": (D + 16, 8), "k": (D + 40, 24), "v": (D + 8, 0), "out": (D + 24, 16), "dout": (D + 32, 8),
                "dq": (D + 16, 0), "dk": (D + 56, 32), "dv": (D + 8, 0)}
        bufs = {nm: _Buf(M, D, pitch, col0, spare=5) for nm, (pitch, col0) in spec.items()}
        for i, nm in enumerate(("q", "k", "v", "dout")):
            bufs[nm].fill(_randn(M, D, seed=60 + i))
        q, k, v, out, dout, dq, dk, dv = (bufs[nm].view for nm in spec)
    lse = _Buf(1, B * H * n, B * H * n + 64, dtype=torch.float32)    # [B, H, n] contiguous, then 64 spare floats
    bufs["lse"] = lse
    kw = _form_kw(form, B, n)
    if form == "keylen":
        _pad_keys(k, v, kw["kv_len"], n, seed=54)
        bufs = {nm: buf for nm, buf in bufs.items() if nm not in ("dqkv", "dq", "dk", "dv")}
    _attn_fwd_raw(q, k, v, out, lse.view, B, n, H, d, scale, form, **kw)
    if form != "keylen":
        _ll().attn_bwd(q, k, v, out, dout, lse.view.reshape(B, H, n), B, n, H, d, scale, dq, dk, dv,
                       causal=kw["causal"], rowscale=kw["rowscale"])
    torch.cuda.synchronize()
    for nm, buf in bufs.items():
        buf.check_poison(nm)
    kept = (torch.ones(B, device="cuda") if form != "plan" else kw["rowscale"][::n]) != 0
    o_ref, lse_ref = attn_ref_fwd(q, k, v, B, n, H, d, scale, causal=kw["causal"], kv_len=kw["kv_len"])
    _tiles("o", out, o_ref * kept.repeat_interleave(n)[:, None], B, n, H, d)
    _lse("lse", lse.view.reshape(B, H, n), lse_ref * kept[:, None, None])
    if form != "keylen":
        refs = attn_ref_bwd(q, k, v, dout, B, n, H, d, scale, causal=kw["causal"])
        for name, got, ref in zip(("dq", "dk", "dv"), (dq, dk, dv), refs):
            _tiles(name, got, ref * kept.repeat_interleave(n)[:, None], B, n, H, d)


# ------------------------------------------------------------------------------------------- bit-exact properties
BITWISE_CASES = [(5, 417, 16, 88), (3, 353, 24, 40), (1, 833, 25, 128)]


def _fwd_bwd(q, k, v, dout, B, n, H, d, scale, causal=False, kv_len=None, rowscale=None):
    """attn_fwd with the form's arguments, then, with dout and without kv_len (no key-length backward), attn_bwd into
    _grad_slots.  Returns (out, lse, (dq, dk, dv) or ())."""
    out, lse = _ll().attn_fwd(q, k, v, B, n, H, d, scale, causal=causal, kv_len=kv_len, rowscale=rowscale)
    if dout is None or kv_len is not None:
        return out, lse, ()
    grads = _grad_slots(B, n, H, d)
    _ll().attn_bwd(q, k, v, out, dout, lse, B, n, H, d, scale, *grads, causal=causal, rowscale=rowscale)
    return out, lse, grads


def _flat(res):
    out, lse, grads = res
    return (out, lse, *grads)


@pytest.mark.parametrize("B,n,H,d,form", _formed(BITWISE_CASES))
def test_attn_bitwise_repeatable(cuda_lib, B, n, H, d, form):
    """One CTA per (row block, head, clip), no atomics, a fixed MMA order: two identical calls give equal bits."""
    q, k, v = _packed(B, n, H, d, seed=71)
    dout = _randn(B * n, H * d, seed=72).to(bf16)
    kw = _form_kw(form, B, n)
    first, second = (_flat(_fwd_bwd(q, k, v, dout, B, n, H, d, d ** -0.5, **kw)) for _ in range(2))
    for name, a, b in zip(("out", "lse", "dq", "dk", "dv"), first, second):
        assert torch.equal(a, b), name


@pytest.mark.parametrize("B,n,H,d,form", _formed(BITWISE_CASES))
def test_attn_items_isolated(cuda_lib, B, n, H, d, form):
    """A (clip, head) item's results equal, bit for bit, those of a B = 1, H = 1 call on views of the same data with
    the same pitches (and that clip's key length or DropPath factor): a CTA's arithmetic depends only on its own item,
    n, d and the scale, so any difference is contamination between items (a stale stage, a barrier phase carried
    over, a wrong head or clip offset)."""
    scale = d ** -0.5
    q, k, v = _packed(B, n, H, d, seed=81)
    dout = _randn(B * n, H * d, seed=82).to(bf16)
    kw = _form_kw(form, B, n)
    out, lse, grads = _fwd_bwd(q, k, v, dout, B, n, H, d, scale, **kw)
    for b, h in {(0, 0), (B - 1, H - 1), (B - 1, 0), (0, H - 1), (B // 2, H // 2)}:
        rows, cols = slice(b * n, (b + 1) * n), slice(h * d, (h + 1) * d)
        one = [t[rows, cols] for t in (q, k, v, dout)]
        kw1 = {"causal": kw["causal"], "kv_len": None if kw["kv_len"] is None else kw["kv_len"][b:b + 1],
               "rowscale": None if kw["rowscale"] is None else kw["rowscale"][rows]}
        o1, l1, g1 = _fwd_bwd(*one, 1, n, 1, d, scale, **kw1)
        assert torch.equal(o1, out[rows, cols]), (b, h, "out")
        assert torch.equal(l1[0, 0], lse[b, h]), (b, h, "lse")
        for name, a, full in zip(("dq", "dk", "dv"), g1, grads):
            assert torch.equal(a, full[rows, cols]), (b, h, name)


# ------------------------------------------------------------------------------------------- exact masking
# A masked key has S = -inf, so its P is exactly 0, and 0 times a finite value is 0: what a mask hides cannot change
# a bit of what it does not.  t: either side of the 64-key tile and the 128-row block, and the last row.
EXACT_N = 190
EXACT_T = (1, 63, 64, 65, 128, 129, EXACT_N - 1)


def _below(B, n, t):
    """bool [B*n, 1]: the rows whose index within their clip is < t."""
    return (torch.arange(B * n, device="cuda") % n < t)[:, None]


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_causal_future_keys_are_exactly_masked(cuda_lib, d):
    """Replacing the K and V rows >= t leaves O, lse and dQ of the rows < t bit for bit unchanged."""
    B, n, H = 2, EXACT_N, 3
    q, k, v = _packed(B, n, H, d, seed=91)
    dout = _randn(B * n, H * d, seed=92).to(bf16)
    k_new, v_new = (_randn(B * n, H * d, seed=93 + i).to(bf16) for i in range(2))
    out, lse, (dq, _, _) = _fwd_bwd(q, k, v, dout, B, n, H, d, d ** -0.5, causal=True)
    for t in EXACT_T:
        keep = _below(B, n, t)
        o2, l2, (dq2, _, _) = _fwd_bwd(q, torch.where(keep, k, k_new), torch.where(keep, v, v_new), dout, B, n, H, d,
                                       d ** -0.5, causal=True)
        rows = keep[:, 0]
        assert torch.equal(o2[rows], out[rows]), (t, "out")
        assert torch.equal(l2[..., :t], lse[..., :t]), (t, "lse")
        assert torch.equal(dq2[rows], dq[rows]), (t, "dq")


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_causal_past_queries_are_exactly_masked(cuda_lib, d):
    """Replacing the Q and dO rows < t leaves O and lse of the rows >= t (the forward run again) and dK and dV of
    the rows >= t bit for bit unchanged."""
    B, n, H = 2, EXACT_N, 3
    q, k, v = _packed(B, n, H, d, seed=94)
    dout = _randn(B * n, H * d, seed=95).to(bf16)
    q_new, dout_new = (_randn(B * n, H * d, seed=96 + i).to(bf16) for i in range(2))
    out, lse, (_, dk, dv) = _fwd_bwd(q, k, v, dout, B, n, H, d, d ** -0.5, causal=True)
    for t in EXACT_T:
        early = _below(B, n, t)
        o2, l2, (_, dk2, dv2) = _fwd_bwd(torch.where(early, q_new, q), k, v, torch.where(early, dout_new, dout), B, n,
                                         H, d, d ** -0.5, causal=True)
        rows = ~early[:, 0]
        assert torch.equal(o2[rows], out[rows]), (t, "out")
        assert torch.equal(l2[..., t:], lse[..., t:]), (t, "lse")
        assert torch.equal(dk2[rows], dk[rows]), (t, "dk")
        assert torch.equal(dv2[rows], dv[rows]), (t, "dv")


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_keylen_padded_keys_are_exactly_masked(cuda_lib, d):
    """One clip per t with kv_len = t: replacing each clip's K and V rows >= kv_len leaves out and lse bit for bit
    unchanged."""
    n, H = EXACT_N, 3
    B = len(EXACT_T)
    kv = torch.tensor(EXACT_T, device="cuda", dtype=torch.int32)
    q, k, v = _packed(B, n, H, d, seed=97)
    k_new, v_new = (_randn(B * n, H * d, seed=98 + i).to(bf16) for i in range(2))
    keep = (torch.arange(B * n, device="cuda") % n < kv.repeat_interleave(n))[:, None]
    out, lse = _ll().attn_fwd(q, k, v, B, n, H, d, d ** -0.5, kv_len=kv)
    o2, l2 = _ll().attn_fwd(q, torch.where(keep, k, k_new), torch.where(keep, v, v_new), B, n, H, d, d ** -0.5,
                            kv_len=kv)
    assert torch.equal(o2, out) and torch.equal(l2, lse)


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_single_key_rows_copy_v(cuda_lib, d):
    """A row with one key has P = exp2(0) = 1 and l = 1, so its O is that key's V row, exactly: causal row 0 of every
    clip, and every row of a clip with kv_len = 1."""
    B, n, H = 3, EXACT_N, 3
    q, k, v = _packed(B, n, H, d, seed=99)
    first = torch.arange(B, device="cuda") * n
    out, _ = _ll().attn_fwd(q, k, v, B, n, H, d, d ** -0.5, causal=True)
    assert torch.equal(out[first], v[first])
    out, _ = _ll().attn_fwd(q, k, v, B, n, H, d, d ** -0.5, kv_len=torch.ones(B, device="cuda", dtype=torch.int32))
    assert torch.equal(out, v[first].repeat_interleave(n, 0))


@pytest.mark.parametrize("n", [40, 77, 129])
@pytest.mark.parametrize("d", [64, 88])
def test_keylen_every_length(cuda_lib, d, n):
    """B = n clips, clip b keeping b + 1 keys: every length from 1 to n in one call, against the reference."""
    B, H = n, 2
    kv = torch.arange(1, n + 1, device="cuda", dtype=torch.int32)
    q, k, v = _packed(B, n, H, d, seed=n + d, scale=1.5)
    _pad_keys(k, v, kv, n, seed=n)
    _check_fwd(q, k, v, B, n, H, d, d ** -0.5, kv_len=kv)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("d", [40, 128])
def test_attn_fwd_without_lse(cuda_lib, d, form):
    """want_lse=False (no lse2 buffer, as the frozen towers call it) gives the out bits of want_lse=True."""
    B, n, H = 3, 353, 4
    q, k, v = _packed(B, n, H, d, seed=d)
    kw = _form_kw(form, B, n)
    out, lse = _ll().attn_fwd(q, k, v, B, n, H, d, d ** -0.5, **kw)
    out2, none = _ll().attn_fwd(q, k, v, B, n, H, d, d ** -0.5, want_lse=False, **kw)
    assert none is None and lse is not None and torch.equal(out2, out)


# ------------------------------------------------------------------------------------------- head-axis attention
@pytest.mark.parametrize("pad", [0, 40])
@pytest.mark.parametrize("d", [64, 88])
@pytest.mark.parametrize("H", [1, 16, 17, 32])
def test_headaxis_attn(cuda_lib, H, d, pad):
    """The VideoMAEv2 teacher's attention as the reference runs it: softmax over the H heads of each token
    (oracle/restate.py:videomae_teacher_forward, head_axis_attention=True).  H <= 16 and 17..32 are two kernel
    instantiations; H = 32 at d = 88 needs more than 48 KB of shared memory.  Pad columns of the qkv pitch are NaN."""
    B, N = 2, 301
    D = H * d
    buf = _Buf(B * N, 3 * D, 3 * D + pad)
    buf.fill(_randn(B * N, 3 * D, seed=H * d))
    qkv = buf.view
    out = _ll().headaxis_attn_fwd(qkv, B, N, H, d, d ** -0.5)
    q, k, v = (qkv[:, i * D:(i + 1) * D].double().reshape(B, N, H, d) for i in range(3))
    s = torch.einsum("btid,btjd->btij", q * d ** -0.5, k)
    o_ref = torch.einsum("btij,btjd->btid", s.softmax(-1), v)                        # [B, N, H, d]
    # the kernel writes [B, H, N, d]; compare token rows with heads as the column blocks
    got = out.permute(0, 2, 1, 3).reshape(B * N, D)
    _tiles("headaxis", got, o_ref.reshape(B * N, D), B, N, H, d)


# ------------------------------------------------------------------------------------------- pool attention
def _pool_ref(q, k, v, dout, B, n, H, d, scale):
    qh = q.double().reshape(B, H, d)
    kh, vh = (t.double().reshape(B, n, H, d) for t in (k, v))
    p = torch.einsum("bhd,bkhd->bhk", qh * scale, kh).softmax(-1)
    o = torch.einsum("bhk,bkhd->bhd", p, vh)
    g = dout.double().reshape(B, H, d)
    dp = torch.einsum("bhd,bkhd->bhk", g, vh)
    ds = p * (dp - (p * dp).sum(-1, keepdim=True))
    dq = scale * torch.einsum("bhk,bkhd->bhd", ds, kh)
    dk = scale * torch.einsum("bhk,bhd->bkhd", ds, qh)
    dv = torch.einsum("bhk,bhd->bkhd", p, g)
    return o.reshape(B, H * d), p, dq.reshape(B, H * d), dk.reshape(B * n, H * d), dv.reshape(B * n, H * d)


# the largest n whose scores fit 48 KB of shared memory: 12280 - d forward, 12280 - 2d backward
POOL_LIMIT_CASES = [(2, 12280 - 88, 4, 88), (2, 12280 - 2 * 88, 4, 88), (1, 12280 - 2 * 128, 2, 128)]


@pytest.mark.parametrize("B,n,H,d", [(2, 417, 16, 88), (3, 13, 2, 64), (1, 1025, 4, 64)] + POOL_LIMIT_CASES)
def test_pool_attention_single_query(cuda_lib, B, n, H, d):
    """AttentionPoolingBlock core: one query per clip (internvideo2_pretrain.py:61-76), k and v in buffers of their
    own."""
    _check_pool(B, n, H, d, slots=False)


@pytest.mark.parametrize("B,n,H,d", [(2, 417, 16, 88), (1, 1025, 4, 64)] + POOL_LIMIT_CASES[:2])
def test_pool_attention_kv_slots(cuda_lib, B, n, H, d):
    """k and v as the middle and last slots of a wider NaN-padded buffer, as the projections of the pooling block
    lay them out."""
    _check_pool(B, n, H, d, slots=True)


def _check_pool(B, n, H, d, slots):
    ll = _ll()
    D = H * d
    scale = d ** -0.5
    q = _randn(B, D, seed=n).to(bf16)
    if slots:
        buf = _Buf(B * n, 3 * D, 3 * D + 16, col0=8)
        buf.fill(_randn(B * n, 3 * D, seed=n + 1))
        k, v = buf.view[:, D:2 * D], buf.view[:, 2 * D:]
    else:
        k, v = _randn(B * n, D, seed=n + 2).to(bf16), _randn(B * n, D, seed=n + 3).to(bf16)
    dout = _randn(B, D, seed=n + 4).to(bf16)
    o_ref, p_ref, dq_ref, dk_ref, dv_ref = _pool_ref(q, k, v, dout, B, n, H, d, scale)
    out, probs = ll.pool_attn_fwd(q, k, v, B, n, H, d, scale)
    _tiles("pool_o", out, o_ref, B, 1, H, d)
    _within("pool_probs", float((probs.double() - p_ref).abs().max()))
    _within("pool_probs_sum", float((probs.double().sum(-1) - 1).abs().max()))
    if n > 12280 - 2 * d:
        with pytest.raises(Exception, match="sequence too long"):
            ll.pool_attn_bwd(q, k, v, probs, dout, B, n, H, d, scale)
        return
    dq, dk, dv = ll.pool_attn_bwd(q, k, v, probs, dout, B, n, H, d, scale)
    _tiles("pool_dq", dq, dq_ref, B, 1, H, d)
    _tiles("pool_dk", dk, dk_ref, B, n, H, d)
    _tiles("pool_dv", dv, dv_ref, B, n, H, d)


def test_flash_attention_module_seam(cuda_lib):
    """The reference's attention seam: FlashAttention()(qkv[B,S,3,H,d]) -> (out[B,S,H,d], None), forward and backward
    (flash_attention_class.py:27-50), plus the refusals for what the pre-training path never passes."""
    from internvideo_b200.patch import FlashAttention
    B, S, H, d = 2, 209, 6, 64
    D = H * d
    qkv = _randn(B, S, 3, H, d, seed=4).to(bf16).requires_grad_(True)
    fa = FlashAttention(attention_dropout=0.0)
    out, none = fa(qkv)
    assert none is None and tuple(out.shape) == (B, S, H, d)
    dout = _randn(B, S, H, d, seed=5).to(bf16)
    out.backward(dout)
    flat = qkv.detach().reshape(B * S, 3 * D)
    q, k, v = flat[:, :D], flat[:, D:2 * D], flat[:, 2 * D:]
    o_ref, _ = attn_ref_fwd(q, k, v, B, S, H, d, d ** -0.5)
    _tiles("o", out.reshape(B * S, D), o_ref, B, S, H, d)
    grads = attn_ref_bwd(q, k, v, dout.reshape(B * S, D), B, S, H, d, d ** -0.5)
    got = qkv.grad.reshape(B * S, 3 * D)
    for i, (name, ref) in enumerate(zip(("dq", "dk", "dv"), grads)):
        _tiles(name, got[:, i * D:(i + 1) * D], ref, B, S, H, d)
    with pytest.raises(NotImplementedError):
        fa(qkv, key_padding_mask=torch.ones(B, S, dtype=torch.bool, device="cuda"))
    with pytest.raises(NotImplementedError):
        fa(qkv, causal=True)
