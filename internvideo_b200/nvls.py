"""Symmetric gradient buffer + the in-switch all-reduce kernel (csrc/ivb_nvls.cu) for the data-parallel engine.

The reference reduces gradients with torch DDP / DeepSpeed over NCCL (run_pretraining.py:378, utils.py:814-834).  Here
the flat bf16 gradient buffer is allocated as SYMMETRIC memory (the same allocation on every rank, peer-mapped and bound
to an NVLink multicast object; torch.distributed._symmetric_memory does the allocation and the handle exchange — plumbing)
and reduced by libivb200's own kernel: `multimem.ld_reduce` / `multimem.st` through the NVSwitch, a handful of CTAs.

    buf = NvlsBuffer(numel, torch.bfloat16, device, group)     # collective
    buf.tensor                                                  # the flat gradient buffer (local view)
    buf.all_reduce_(start, end)                                 # collective, on the current stream; sum over ranks

Raises NvlsUnavailable when the platform cannot do it (one rank, no multicast support, handle exchange refused): the
engine then keeps NCCL.  There is no silent fallback inside all_reduce_() itself.
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

from . import _lib
from . import lowlevel as ll


class NvlsUnavailable(RuntimeError):
    pass


def default_blocks(world: int = 8) -> int:
    """CTAs per reduction.  A rank pulls 1/world of every range through the switch, so small worlds need more requests in
    flight per rank: 16 CTAs below 4 GPUs, else 8 (IVB_NVLS_BLOCKS overrides).  Not measured on H100."""
    env = os.environ.get("IVB_NVLS_BLOCKS")
    if env:
        return int(env)
    return 16 if world < 4 else 8


class NvlsBuffer:
    def __init__(self, numel: int, dtype, device, group=None, nblocks: int | None = None):
        if not dist.is_initialized():
            raise NvlsUnavailable("torch.distributed is not initialised")
        group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        if self.world < 2 or self.world > 16:
            raise NvlsUnavailable(f"world size {self.world} (needs 2..16 ranks on one NVSwitch domain)")
        if dtype != torch.bfloat16:
            raise NvlsUnavailable("only bf16 gradients are reduced in the switch")
        device = torch.device(device)
        if device.type != "cuda":
            raise NvlsUnavailable("not a CUDA device")
        try:
            import torch.distributed._symmetric_memory as symm_mem
            from torch._C._distributed_c10d import _SymmetricMemory
        except Exception as e:                                    # pragma: no cover
            raise NvlsUnavailable(f"torch symmetric memory is not available: {e}")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        try:
            from torch._C._autograd import DeviceType
            if not _SymmetricMemory.has_multicast_support(DeviceType.CUDA, idx):
                raise NvlsUnavailable("the driver / fabric reports no NVLink multicast support")
            words = _lib.load().ivb_nvls_flag_words()
            self.tensor = symm_mem.empty(numel, dtype=dtype, device=device)
            self.tensor.zero_()
            self.flags = symm_mem.empty(words, dtype=torch.int32, device=device)
            self.flags.zero_()
            torch.cuda.synchronize(device)
            self.hdl = symm_mem.rendezvous(self.tensor, group)
            self.flag_hdl = symm_mem.rendezvous(self.flags, group)
        except NvlsUnavailable:
            raise
        except Exception as e:
            raise NvlsUnavailable(f"symmetric allocation / rendezvous failed: {type(e).__name__}: {e}")
        self.mc_ptr = int(self.hdl.multicast_ptr)
        if self.mc_ptr == 0:
            raise NvlsUnavailable("rendezvous returned no multicast address")
        self.flag_ptrs_dev = int(self.flag_hdl.buffer_ptrs_dev)
        self.nblocks = nblocks if nblocks is not None else default_blocks(self.world)
        self.numel = numel
        self.flag_hdl.barrier()          # every rank's flags are zero before anybody signals

    def all_reduce_(self, start: int = 0, end: int | None = None, wide: bool = False):
        """Sum elements [start, end) over the ranks, in place on every rank, on the current CUDA stream.
        wide: four times the CTAs (the caller knows nothing else is competing for the SMs)."""
        end = self.numel if end is None else end
        end = min((end + 7) // 8 * 8, self.numel)      # entries are 16-byte aligned; the pad between them is nobody's
        rc = _lib.load().ivb_nvls_allreduce_bf16(self.mc_ptr, start, end - start, self.flag_ptrs_dev, self.rank,
                                                 self.world, min(self.nblocks * 4, 64) if wide else self.nblocks, ll._stream())
        _lib.check(rc, "ivb_nvls_allreduce_bf16")
