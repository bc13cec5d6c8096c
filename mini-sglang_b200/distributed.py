"""Tensor-parallel communication plug-in: a one-shot NVLink all-reduce (optionally fused with the
residual add + RMSNorm that follows) behind the reference's own plug-in point.

The reference routes every TP collective through ``DistributedCommunicator.plugins[-1]``
(``python/minisgl/distributed/impl.py:60-68``) and installs its capturable NCCL wrapper with
``enable_pynccl_distributed`` (impl.py:71-90).  :func:`enable_b200_allreduce` appends
:class:`B200DistributedImpl` the same way: decode-sized ``all_reduce`` calls (one per layer after
``o_proj`` and after ``down_proj``, layers/linear.py:102-106,122-126 -- inside the captured decode
graphs) run the sm_90a push kernel of ``csrc/allreduce.cu``; larger messages (prefill) and
``all_gather`` are handed to the plug-in that was active before (the reference's NCCL), as
north_star keeps it.

Set-up uses ``torch.distributed`` only to exchange the 64-byte CUDA IPC handles of the per-rank
regions; the data path is hand-written (16-byte peer stores over NVLink; the payload is its own
arrival flag, see csrc/allreduce.cu).
"""

from __future__ import annotations

import ctypes as C
from typing import List, Optional

import torch

from . import _cabi

_DTYPE_CODE = {torch.bfloat16: 0, torch.float16: 1}
DEFAULT_MAX_BYTES = 1 << 20  # 512 rows x 1024 x bf16; decode messages of every BASELINE config fit


class B200AllReduce:
    """One communicator per TP group and device.  ``group`` is any ``torch.distributed`` group that
    contains exactly the TP ranks (gloo or nccl: only ``all_gather_object`` / ``barrier`` are used)."""

    def __init__(self, rank: int, world: int, group, device: torch.device, max_bytes: int = DEFAULT_MAX_BYTES):
        if not (1 <= world <= 8 and 0 <= rank < world):
            raise ValueError(f"bad rank/world {rank}/{world} (world <= 8)")
        self.rank, self.world, self.group = rank, world, group
        self.device = torch.device(device)
        self._lib = _cabi.load()
        self._comm = C.c_void_p()
        with torch.cuda.device(self.device):
            nbytes = self._lib.b200_ar_region_bytes(world, max_bytes)
            local = C.c_void_p()
            _cabi.check(self._lib.b200_ar_alloc(nbytes, C.byref(local)), "b200_ar_alloc")
            handle = (C.c_ubyte * 64)()
            _cabi.check(self._lib.b200_ar_ipc_handle(local, handle), "b200_ar_ipc_handle")
            handles: List[Optional[bytes]] = [None] * world
            torch.distributed.all_gather_object(handles, bytes(handle), group=group)
            bases = (C.c_void_p * world)()
            opened = (C.c_int * world)()
            for i, h in enumerate(handles):
                if i == rank:
                    bases[i] = local.value
                    continue
                buf = (C.c_ubyte * 64).from_buffer_copy(h)
                peer = C.c_void_p()
                _cabi.check(self._lib.b200_ar_ipc_open(buf, C.byref(peer)), f"b200_ar_ipc_open(rank {i})")
                bases[i], opened[i] = peer.value, 1
            _cabi.check(
                self._lib.b200_ar_create(rank, world, bases, opened, max_bytes, C.byref(self._comm)), "b200_ar_create"
            )
        self.max_bytes = int(self._lib.b200_ar_max_bytes(self._comm))
        torch.distributed.barrier(group=group)  # every rank has mapped every region before the first push

    def fits(self, x: torch.Tensor) -> bool:
        """True when the kernel accepts a contiguous ``x``: anything else goes to the fallback."""
        return x.is_cuda and x.dtype in _DTYPE_CODE and x.dim() >= 1 and x.shape[-1] % 8 == 0 and \
            x.data_ptr() % 16 == 0 and x.numel() * x.element_size() <= self.max_bytes

    def all_reduce(self, x: torch.Tensor, out: Optional[torch.Tensor] = None,
                   residual: Optional[torch.Tensor] = None, weight: Optional[torch.Tensor] = None,
                   eps: float = 0.0) -> torch.Tensor:
        """``out <- sum over ranks of x`` (in place when ``out`` is None).  With ``residual`` and
        ``weight``: ``residual += sum`` and ``out <- rmsnorm(residual) * weight`` (the semantics of
        the all-reduce followed by ``fused_add_rmsnorm``, one launch)."""
        if self._comm.value is None:
            raise RuntimeError("B200AllReduce was destroyed")
        if not x.is_cuda:
            raise RuntimeError("B200AllReduce needs CUDA tensors (no CPU path)")
        x2 = x.view(-1, x.shape[-1])
        o2 = x2 if out is None else out.view(-1, out.shape[-1])
        if x2.stride(1) != 1 or o2.stride(1) != 1 or o2.shape != x2.shape or o2.dtype != x2.dtype:
            raise RuntimeError("all_reduce: x / out must be matching row-major 2-D views")
        if (residual is None) != (weight is None):
            raise RuntimeError("all_reduce: residual and weight go together")
        r2 = None
        if residual is not None:
            r2 = residual.view(-1, residual.shape[-1])
            if r2.shape != x2.shape or r2.dtype != x2.dtype or r2.stride(1) != 1 or weight.shape != (x2.shape[1],) \
                    or weight.dtype != x2.dtype or not weight.is_contiguous():
                raise RuntimeError("all_reduce: residual / weight shape or dtype mismatch")
        code = _DTYPE_CODE.get(x2.dtype)
        if code is None:
            raise RuntimeError(f"all_reduce: unsupported dtype {x2.dtype}")
        _cabi.check(
            self._lib.b200_ar_allreduce(
                self._comm, x2.data_ptr(), x2.stride(0), o2.data_ptr(), o2.stride(0),
                r2.data_ptr() if r2 is not None else None, r2.stride(0) if r2 is not None else 0,
                weight.data_ptr() if weight is not None else None, x2.shape[0], x2.shape[1], float(eps),
                code, torch.cuda.current_stream(x.device).cuda_stream,
            ),
            "b200_ar_allreduce",
        )
        return x if out is None else out

    def destroy(self) -> None:
        if self._comm.value is not None:
            torch.cuda.synchronize(self.device)
            torch.distributed.barrier(group=self.group)  # nobody unmaps while a peer may still push
            self._lib.b200_ar_destroy(self._comm, 1)
            self._comm = C.c_void_p()


class B200DistributedImpl:
    """``DistributedImpl`` (reference distributed/impl.py:16-21) whose ``all_reduce`` uses the push
    kernel when the message fits and otherwise defers to ``fallback`` -- the plug-in that was active
    before (the reference's NCCL path), not a CPU path."""

    def __init__(self, comm: B200AllReduce, fallback) -> None:
        self.comm = comm
        self.fallback = fallback

    def all_reduce(self, x: torch.Tensor) -> torch.Tensor:
        if self.comm.fits(x) and x.is_contiguous():
            return self.comm.all_reduce(x)
        return self.fallback.all_reduce(x)

    def all_gather(self, x: torch.Tensor) -> torch.Tensor:
        return self.fallback.all_gather(x)


def enable_b200_allreduce(tp_rank: int, tp_size: int, tp_cpu_group, device, max_bytes: int = DEFAULT_MAX_BYTES):
    """Append the plug-in to the reference's ``DistributedCommunicator.plugins`` (call after
    ``Engine`` has set up its own communication, engine/engine.py:117-139).  Returns the
    communicator, or None for tp_size 1."""
    if tp_size == 1:
        return None
    from minisgl.distributed import DistributedCommunicator

    comm = B200AllReduce(tp_rank, tp_size, tp_cpu_group, device, max_bytes)
    DistributedCommunicator.plugins.append(B200DistributedImpl(comm, DistributedCommunicator.plugins[-1]))
    return comm
