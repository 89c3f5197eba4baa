"""The attention entry points refuse bad arguments before touching the device, so their refusals are checked here
through the raw C ABI with null pointers: each returns non-zero with its message in ivb_last_error(), and an empty
batch or sequence is a no-op that returns 0."""
import pytest

from abi_fake import expect_refusal
from internvideo_b200 import _lib

D16 = 16 * 88


def _fwd(lib, d=88, H=16, ld=(3 * D16, 3 * D16, 3 * D16, D16), B=2, n=417):
    return lib.ivb_attn_fwd(None, ld[0], None, ld[1], None, ld[2], None, ld[3], None, B, n, H, d, 0.1, None)


def _bwd(lib, d=88, H=16, ld=(3 * D16,) * 3 + (D16,) * 2 + (3 * D16,) * 3, B=2, n=417, lse=1, ws=1024):
    return lib.ivb_attn_bwd(None, ld[0], None, ld[1], None, ld[2], None, ld[3], None, ld[4], lse, ws,
                            None, ld[5], None, ld[6], None, ld[7], B, n, H, d, 0.1, None)


@pytest.mark.parametrize("d", [8, 12, 136, 0, -8])
def test_attn_head_dim_refused(d):
    lib = _lib.load()
    expect_refusal(_fwd(lib, d=d), "ivb_attn_fwd: head_dim must be a multiple of 8 in [16,128]")
    expect_refusal(_bwd(lib, d=d), "ivb_attn_bwd: head_dim must be a multiple of 8 in [16,128]")


@pytest.mark.parametrize("slot", range(8))
def test_attn_pitch_refused(slot):
    lib = _lib.load()
    ld = [3 * D16] * 3 + [D16] * 2 + [3 * D16] * 3
    ld[slot] += 4
    expect_refusal(_bwd(lib, ld=ld), "ivb_attn_bwd: pitches must be multiples of 8")
    if slot < 4:
        expect_refusal(_fwd(lib, ld=ld[:4]), "ivb_attn_fwd: pitches must be multiples of 8")


def test_attn_bwd_workspace_refused():
    lib = _lib.load()
    expect_refusal(_bwd(lib, lse=None), "ivb_attn_bwd: lse2 and the workspace are required")
    expect_refusal(_bwd(lib, ws=None), "ivb_attn_bwd: lse2 and the workspace are required")
    expect_refusal(_bwd(lib, ws=1032), "ivb_attn_bwd: workspace must be 16-byte aligned")


def test_attn_empty_is_a_noop():
    lib = _lib.load()
    for B, n in ((0, 417), (2, 0), (0, 0)):
        assert _fwd(lib, B=B, n=n) == 0
        assert _bwd(lib, B=B, n=n) == 0
        assert lib.ivb_headaxis_attn_fwd(None, 3 * D16, B, n, 16, 88, 0.1, None, None) == 0
    assert lib.ivb_pool_attn_fwd(None, None, D16, None, D16, 0, 417, 16, 88, 0.1, None, None, None) == 0
    assert lib.ivb_pool_attn_bwd(None, None, D16, None, D16, None, None, 0, 417, 16, 88, 0.1,
                                 None, None, D16, None, D16, None) == 0


@pytest.mark.parametrize("H", [0, 33])
def test_headaxis_heads_refused(H):
    lib = _lib.load()
    expect_refusal(lib.ivb_headaxis_attn_fwd(None, 3 * H * 64, 2, 1568, H, 64, 0.125, None, None),
                   "ivb_headaxis_attn_fwd: 1 <= heads <= 32")


@pytest.mark.parametrize("d,ld", [(12, 3 * 16 * 16), (64, 3 * 16 * 64 + 4)])
def test_headaxis_head_dim_and_pitch_refused(d, ld):
    lib = _lib.load()
    expect_refusal(lib.ivb_headaxis_attn_fwd(None, ld, 2, 1568, 16, d, 0.1, None, None),
                   "ivb_headaxis_attn_fwd: head_dim / pitch must be multiples of 8")


@pytest.mark.parametrize("d,ldk,ldv", [(12, D16, D16), (88, D16 + 4, D16), (88, D16, D16 + 2)])
def test_pool_head_dim_and_pitch_refused(d, ldk, ldv):
    lib = _lib.load()
    expect_refusal(lib.ivb_pool_attn_fwd(None, None, ldk, None, ldv, 2, 417, 16, d, 0.1, None, None, None),
                   "ivb_pool_attn_fwd: d/ld must be multiples of 8")
    expect_refusal(lib.ivb_pool_attn_bwd(None, None, ldk, None, ldv, None, None, 2, 417, 16, d, 0.1,
                                         None, None, D16, None, D16, None),
                   "ivb_pool_attn_bwd: d/ld must be multiples of 8")
    expect_refusal(lib.ivb_pool_attn_bwd(None, None, D16, None, D16, None, None, 2, 417, 16, 88, 0.1,
                                         None, None, D16 + 4, None, D16, None),
                   "ivb_pool_attn_bwd: d/ld must be multiples of 8")


@pytest.mark.parametrize("d", [64, 88, 128])
def test_pool_sequence_limit_refused(d):
    """The scores of one (clip, head) must fit 48 KB of shared memory: n <= 12280 - d forward, 12280 - 2d backward."""
    lib = _lib.load()
    expect_refusal(lib.ivb_pool_attn_fwd(None, None, D16, None, D16, 2, 12280 - d + 1, 16, d, 0.1, None, None, None),
                   "ivb_pool_attn_fwd: sequence too long for the single-query kernel")
    expect_refusal(lib.ivb_pool_attn_bwd(None, None, D16, None, D16, None, None, 2, 12280 - 2 * d + 1, 16, d, 0.1,
                                         None, None, D16, None, D16, None),
                   "ivb_pool_attn_bwd: sequence too long for the single-query kernel")
