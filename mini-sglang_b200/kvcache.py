"""Paged KV pool with the reference's interface (``BaseKVCachePool`` / ``MHAKVCache``,
``python/minisgl/kvcache/base.py:10-38``, ``mha_pool.py:10-68``).

Inside mini-sglang the engine's own pool is borrowed as is (same layout); this class exists so the
backend, the tests and ``bench.py`` can run where the reference is not installed, and so that
``store_kv`` goes through the sm_90a store kernel.

HBM layout (identical to the reference): one tensor ``[2, L, num_pages, page_size, Hkv_local, D]``;
``k_cache(l)`` / ``v_cache(l)`` are the contiguous ``[num_pages, page_size, Hkv_local, D]`` slices;
a token slot ``s = page * page_size + offset`` addresses the row ``[s // page_size, s % page_size]``,
i.e. row ``s`` of the ``[num_pages * page_size, Hkv_local * D]`` view the kernels use.
"""

from __future__ import annotations

import torch

from .ops import store_cache
from .utils import div_even, get_tp_info


class MHAKVCache:
    def __init__(
        self,
        num_kv_heads: int,
        num_layers: int,
        head_dim: int,
        num_pages: int,
        page_size: int,
        dtype: torch.dtype,
        device: torch.device,
    ) -> None:
        local_kv_heads = div_even(num_kv_heads, get_tp_info().size, allow_replicate=True)
        self._kv_buffer = torch.empty(
            (2, num_layers, num_pages, page_size, local_kv_heads, head_dim),
            device=device,
            dtype=dtype,
        )
        self._num_layers = num_layers
        self._device = torch.device(device)
        self._rows = num_pages * page_size
        self._row_shape = (self._rows, local_kv_heads, head_dim)

    def k_cache(self, index: int) -> torch.Tensor:
        return self._kv_buffer[0, index]

    def v_cache(self, index: int) -> torch.Tensor:
        return self._kv_buffer[1, index]

    def store_kv(self, k: torch.Tensor, v: torch.Tensor, out_loc: torch.Tensor, layer_id: int) -> None:
        store_cache(
            k_cache=self._kv_buffer[0, layer_id].view(self._row_shape),
            v_cache=self._kv_buffer[1, layer_id].view(self._row_shape),
            indices=out_loc,
            k=k,
            v=v,
        )

    @property
    def device(self) -> torch.device:
        return self._device

    @property
    def dtype(self) -> torch.dtype:
        return self._kv_buffer.dtype

    @property
    def num_layers(self) -> int:
        return self._num_layers
