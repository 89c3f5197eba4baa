"""Both profilers see the library calls of a training block through the one call path: OpProfiler every call, in call
order; GemmProfiler exactly the tensor-core calls and the casts that feed them, with their flop counts."""
import pytest
import torch

from internvideo_b200 import _lib
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import modules as M

pytestmark = pytest.mark.gpu

B, N_TOK, D, H = 4, 257, 128, 2          # B * n >= 1024 rows: the fused RMSNorm + LayerScale backward runs
HOST_QUERIES = {"ivb_attn_bwd_workspace_floats"}     # library calls that launch nothing and take no stream
GEMM_KINDS = {"gemm_bf16": "gemm", "gemm_fp8": "gemm", "attn_fwd": "attn_fwd", "attn_bwd": "attn_bwd",
              "fp8_quantize": "fp8_quantize", "fp8_quantize_rows": "fp8_quantize", "norm_fwd_fp8": "norm_fwd_fp8"}


class _LoggingLib:
    """Stands in for the loaded CDLL and logs each ivb_* call with its arguments."""

    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self.lib, name)

        def logged(*args):
            self.calls.append((name, args))
            return fn(*args)
        return logged


def _block_step():
    """One bf16 RMSNorm block forward and backward with q/k norms, LayerScale and DropPath row scales."""
    torch.manual_seed(0)
    blk = M.Block(D, H, 4, init_values=0.1, qk_normalization=True).bfloat16().cuda()
    x = torch.randn(B * N_TOK, D, device="cuda").requires_grad_(True)
    keep = torch.tensor([1.25, 0.0, 1.25, 1.25], device="cuda").repeat_interleave(N_TOK)
    y = blk.forward_stream(x, B, N_TOK, rowscale=(keep, keep))
    y.backward(torch.randn_like(y))
    torch.cuda.synchronize()


def _profile(prof, monkeypatch):
    _block_step()                                                  # warm-up: module loads, shared-memory limits
    log = _LoggingLib(_lib.load())
    monkeypatch.setattr(_lib, "_lib", log)
    prof.enable()
    try:
        _block_step()
    finally:
        prof.disable()
    return [(name[len("ivb_"):], args) for name, args in log.calls if name not in HOST_QUERIES]


def test_op_profiler_records_every_library_call(cuda_lib, monkeypatch):
    prof = ll.OpProfiler()
    calls = _profile(prof, monkeypatch)
    names = [r[0] for r in prof.records]
    assert [n if not n.startswith("gemm[") else "gemm_bf16" for n in names] == [c for c, _ in calls]
    assert {"rmsnorm_pair_fwd", "rmsnorm_pair_bwd", "rmsnorm_bwd_layerscale"} <= set(names)
    for n, (count, ms) in prof.summary():
        assert count >= 1 and ms >= 0.0, n


def test_gemm_profiler_records_the_tensor_core_calls(cuda_lib, monkeypatch):
    prof = ll.GemmProfiler()
    calls = _profile(prof, monkeypatch)
    assert [r[1] for r in prof.records] == [GEMM_KINDS[c] for c, _ in calls if c in GEMM_KINDS]
    gemms = [args for c, args in calls if c == "gemm_bf16"]
    flops, _ = prof.totals("gemm")
    assert flops == sum(2.0 * M_ * N_ * K_ for M_, N_, K_ in (a[6:9] for a in gemms)) and prof.count == len(gemms)
    assert prof.totals("attn_fwd")[0] == 4.0 * B * H * N_TOK * N_TOK * (D // H)
    assert prof.totals("attn_bwd")[0] == 10.0 * B * H * N_TOK * N_TOK * (D // H)
