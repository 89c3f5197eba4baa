"""DropPath plans (ivb_droppath_plan, ivb_gemm_bf16_plan): the liveness rules, restated in tests/droppath_ref.py, give
the tile order, live count and k-block list that clip-level reasoning predicts for the draws the recipe can make; and
the GEMM refuses a plan it cannot run before any CUDA call."""
import numpy as np
import pytest

from internvideo_b200 import _lib
import droppath_ref as ref
from abi_fake import BASE, cpu_only, expect_refusal

B = 32
DRAWS = {
    "none_dropped": np.ones(B, bool),
    "all_dropped": np.zeros(B, bool),
    "single_clip": np.arange(B) == 5,
    "alternating": np.arange(B) % 2 == 0,
}


def _expected(keep, n):
    """Tiles and k-blocks that overlap a kept clip's rows [b n, (b + 1) n)."""
    M = keep.size * n
    def live(size, count):
        return [i for i in range(count) if any(keep[b] and b * n < (i + 1) * size and i * size < (b + 1) * n
                                               for b in range(keep.size))]
    return live(128, (M + 127) // 128), live(64, (M + 63) // 64)


@pytest.mark.parametrize("n", [417, 65, 256])
@pytest.mark.parametrize("draw", list(DRAWS))
def test_plan_matches_clip_liveness(draw, n):
    keep = DRAWS[draw]
    M = B * n
    order, live, klist = ref.plan(ref.clip_rows(keep, n))
    tiles, kbs = _expected(keep, n)
    nm = (M + 127) // 128
    assert sorted(order) == list(range(nm))
    assert order[:live] == tiles and live == len(tiles)
    assert order[live:] == sorted(set(range(nm)) - set(tiles))
    assert klist == kbs
    if draw == "none_dropped":
        assert order == list(range(nm)) and live == nm and klist == list(range((M + 63) // 64))
    if draw == "all_dropped":
        assert live == 0 and klist == []
    assert len(ref.flat(order, live, klist, M)) == _lib.load().ivb_droppath_plan_ints(M)


def test_tile_live_when_any_row_kept():
    """A tile is live when one row of it is kept, whichever: the last row of the matrix's ragged tile, or one row of
    a tile otherwise dropped."""
    rs = np.zeros(417, np.float32)
    rs[416] = 2.0
    assert ref.plan(rs) == ([3, 0, 1, 2], 1, [6])
    rs[:] = 0
    rs[200] = 1.0
    assert ref.plan(rs) == ([1, 0, 2, 3], 1, [3])


# ---- refusals, through the raw C ABI with fake device addresses (never reach a launch: CPU-only)
EPI_BF16, EPI_F32, EPI_RESID = 0, 1, 3
FLAG_ACCUM, FLAG_2CTA = 2, 8


def _call(a_mn=0, b_mn=0, epi=EPI_BF16, flags=0, bias=None, m_plan=None, k_plan=None, aux=None):
    M, N, K = 1024, 512, 1024
    return _lib.load().ivb_gemm_bf16_plan(BASE + 0x100000, a_mn, M if a_mn else K, BASE + 0x200000, b_mn,
                                          N if b_mn else K, M, N, K, epi, flags, BASE, N, None, 0, bias, None, aux,
                                          N if aux else 0, None, 0, m_plan, k_plan, None)


@cpu_only
@pytest.mark.parametrize("kw, text", [
    (dict(flags=FLAG_2CTA, m_plan=BASE + 0x300000), "a DropPath plan needs a single-CTA kernel"),
    (dict(a_mn=1, b_mn=1, flags=FLAG_2CTA, k_plan=BASE + 0x300000), "a DropPath plan needs a single-CTA kernel"),
    (dict(flags=FLAG_ACCUM, m_plan=BASE + 0x300000), "an M plan excludes IVB_FLAG_ACCUM"),
    (dict(k_plan=BASE + 0x300000), "a K plan needs both operands MN-major"),
    (dict(a_mn=1, b_mn=1, bias=BASE + 0x400000, k_plan=BASE + 0x300000), "a K plan needs IVB_EPI_BF16 or IVB_EPI_F32"),
    (dict(a_mn=1, b_mn=1, epi=EPI_RESID, aux=BASE + 0x400000, k_plan=BASE + 0x300000),
     "a K plan needs IVB_EPI_BF16 or IVB_EPI_F32"),
])
def test_gemm_refuses_a_plan_it_cannot_run(kw, text):
    expect_refusal(_call(**kw), text)


def test_fp8_gemm_takes_no_plan():
    """The FP8 GEMMs keep their unplanned path: neither the C entry point nor its binding has a plan argument."""
    from internvideo_b200 import lowlevel as ll
    import inspect
    assert len(_lib.PROTOTYPES["ivb_gemm_fp8"][1]) == 25
    assert not {"m_plan", "k_plan"} & set(inspect.signature(ll.gemm_fp8).parameters)
