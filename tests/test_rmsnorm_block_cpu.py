"""The slice check of tests/test_rmsnorm_block_gpu.py's end-to-end comparison (tests/local_err.py with its LOCAL bounds):
an error confined to one token row, one weight-gradient channel or one q/k-norm head, twice the slice bound, stays under
the per-tensor bound, and the slice check catches it and names the slice; the same tensors without it pass both."""
import pytest
import torch

from local_err import rel, slice_errors, worst_slice
from test_rmsnorm_block_gpu import LOCAL

# (LOCAL key, shape of the synthetic result, slices, per-tensor bound, the slice that carries the error)
CASES = {
    "token_row": ("branch_row", (834, 384), 834, 1e-2, 417),
    "dx_row": ("dx_row", (834, 384), 834, 1e-2, 416),
    "qkv_channel": ("attn.qkv.weight", (1152, 384), 1152, 3e-2, 700),
    "fc2_channel": ("mlp.fc2.weight", (384, 1536), 384, 3e-2, 0),
    "q_norm_head": ("attn.q_norm.weight", (384,), 6, 3e-2, 4),
    "k_norm_head": ("attn.k_norm.weight", (1600,), 25, 3e-2, 24),
}


@pytest.mark.parametrize("case", list(CASES))
def test_slice_check_catches_an_error_the_tensor_norm_hides(case):
    key, shape, slices, tensor_bound, bad = CASES[case]
    g = torch.Generator().manual_seed(7)
    ref = torch.randn(shape, generator=g, dtype=torch.float64)
    got = ref * (1 + 1e-3 * torch.randn(shape, generator=g, dtype=torch.float64))   # a correct result's rounding
    assert rel(got, ref) < tensor_bound
    e, _ = worst_slice(slice_errors(got, ref, slices))
    assert e <= LOCAL[key]

    flat = got.reshape(slices, -1)
    step = torch.randn(flat.shape[1], generator=g, dtype=torch.float64)
    typical = float(ref.norm()) / slices ** 0.5
    flat[bad] += 2 * LOCAL[key] * typical * step / step.norm()
    assert rel(got, ref) < tensor_bound, "the confined error must pass the per-tensor bound"
    e, where = worst_slice(slice_errors(got, ref, slices))
    assert e > LOCAL[key] and where == bad, (e, where)


def test_slice_errors_ignore_a_small_reference_slice():
    """A slice whose reference is 1/100 of the others, with an error the size of a correct result's rounding relative to
    the tensor, is not read as a large error."""
    g = torch.Generator().manual_seed(8)
    ref = torch.randn((64, 256), generator=g, dtype=torch.float64)
    ref[3] *= 0.01
    got = ref + 1e-3 * ref.norm() / 64 ** 0.5 / 256 ** 0.5 * torch.randn((64, 256), generator=g, dtype=torch.float64)
    e, _ = worst_slice(slice_errors(got, ref, 64))
    assert e < 2e-3
