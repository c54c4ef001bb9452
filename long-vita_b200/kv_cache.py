"""K/V cache for incremental decoding (SURVEY.md 8f-2).

The reference's Megatron serving loop re-runs the whole prefill for every generated token
(long_vita_megatron/inference/text_generation/generation.py:127-135: with `use_kv_cache` off the full
`tokens` are fed each step) - O(S^2) per token.  Its HF path delegates the cache to transformers'
`DynamicCache` (modeling_long_vita.py:150-151), which grows by `torch.cat` and so re-copies the whole
cache every step.  Here the cache is one pre-allocated [capacity, hkv, d] bf16 buffer per layer for K and
for V, holding post-RoPE rows; a step appends one row per layer and the decode attention reads each row
once (`ops.attention_decode`).

Duck-types the part of transformers' `Cache` the reference touches: `len(cache)` (`modeling_long_vita.py:90`)
and `get_seq_length()` (:154).

Rows appended by a forward pass are pending until it ends: `commit()` when one call runs every layer (run_layers),
`commit_to(offset)` under Megatron's `--use-kv-cache` protocol, where each layer is a call of its own and
`inference_params.sequence_len_offset` says how many tokens earlier forwards have written.

A cache that does not fit in HBM beside the prefill is an `OffloadedKVCache`: its leading layers are the device
buffers above, the others one pinned host buffer each, read in place by the decode kernel (`ops.attention_decode_host`).
`make_cache` decides which, once, from the free device memory (`device_layers`).

The host tier may be kept in FP8 (`host_dtype=torch.float8_e4m3fn`): e4m3 K|V rows with one fp32 scale per head
(csrc/fp8_core.h), 2112 instead of 4096 bytes per row at 8 kv heads, which halves both the pinned memory and the
PCIe bytes a decode step reads.  It is lossy and opt-in; the default is bf16, and the device layers are bf16 either way.

Several questions about one prompt (a long video) share its cache as a `ContextCache`: the filled cache of the
prompt, never written again.  Each question runs in a `ContextSession`, the context plus a private device `KVCache`
suffix for the question's and the answer's rows, so that a question costs a prefill of its own tokens only.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from . import ops


class KVCache:
    def __init__(self, num_layers: int, capacity: int, num_kv_heads: int, head_dim: int, device, dtype=torch.bfloat16):
        self.capacity = int(capacity)
        self.k: List[torch.Tensor] = [torch.empty((self.capacity, num_kv_heads, head_dim), dtype=dtype, device=device)
                                      for _ in range(num_layers)]
        self.v: List[torch.Tensor] = [torch.empty((self.capacity, num_kv_heads, head_dim), dtype=dtype, device=device)
                                      for _ in range(num_layers)]
        self._len = 0            # tokens whose K/V rows are valid in EVERY layer
        self._pending = 0        # rows appended by the forward pass in flight (committed at its end)

    def __len__(self) -> int:
        return self._len

    def get_seq_length(self, layer_idx: int = 0) -> int:
        return self._len

    def append(self, layer_idx: int, k: torch.Tensor, v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, int]:
        """Write k / v [t, hkv, d] behind the committed rows of `layer_idx`; returns (K, V, new_length)
        where K / V are the cache buffers (valid rows [0, new_length))."""
        t = k.shape[0]
        end = self._len + t
        if end > self.capacity:
            raise RuntimeError(f"KV cache overflow: {end} tokens > capacity {self.capacity}")
        self.k[layer_idx][self._len : end].copy_(k)
        self.v[layer_idx][self._len : end].copy_(v)
        self._pending = t
        return self.k[layer_idx], self.v[layer_idx], end

    def commit(self) -> None:
        """Called once per forward pass, after the last layer."""
        self._len += self._pending
        self._pending = 0

    def commit_to(self, offset: int) -> None:
        _commit_to(self, offset)

    def bytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self.k + self.v)


def _commit_to(cache, offset: int) -> None:
    """Megatron's protocol: a forward starts with `offset` (inference_params.sequence_len_offset) tokens written by
    earlier forwards, and Megatron advances the offset by the forward's length after it.  So an offset equal to the
    committed length is this forward (its first layer, or a later one with rows pending), and an offset that moved by
    exactly the pending rows starts the next forward: those rows are committed first.  Anything else (the offset moved
    back, or past the pending rows) cannot come from that protocol and raises, with the cache unchanged."""
    offset = int(offset)
    if cache._pending and offset == cache._len + cache._pending:
        cache.commit()
    elif offset != cache._len:
        raise ValueError(f"K/V cache: sequence_len_offset {offset} does not follow the cache ({cache._len} tokens "
                         f"committed, {cache._pending} pending)")


# Device memory a forward with a K/V cache leaves free beside the cache and the prefill's per-token working set: the
# vision phase's activations, the logits, RoPE and index tensors, the caching allocator's slack.
KV_RESERVE = 4 << 30


def device_free_bytes(device) -> Optional[int]:
    """Device memory a new cache may take on `device`: free memory plus what PyTorch's allocator holds unused; None
    for a device without a memory budget (a CPU tensor cache)."""
    device = torch.device(device)
    if device.type != "cuda":
        return None
    free, _ = torch.cuda.mem_get_info(device)
    return free + torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)


def device_layers(free_bytes: Optional[int], capacity: int, num_layers: int, kv_row_bytes: int, prefill_bytes: int,
                  offloaded_prefill_bytes: int, reserve: int = KV_RESERVE) -> int:
    """How many leading layers of a cache of `capacity` rows (`kv_row_bytes` of K and V per row and layer) stay on
    the device.  `num_layers` - the plain KVCache - when the whole cache, the prefill's device working set
    `prefill_bytes` and `reserve` fit in `free_bytes` (None: no budget); otherwise as many as fit beside the working
    set of the prefill with the cache offloaded, `offloaded_prefill_bytes`, and at most num_layers - 1."""
    layer = capacity * kv_row_bytes
    if free_bytes is None or num_layers * layer + prefill_bytes + reserve <= free_bytes:
        return num_layers
    return int(max(0, min(num_layers - 1, (free_bytes - offloaded_prefill_bytes - reserve) // layer)))


HOST_DTYPES = (torch.bfloat16, torch.float8_e4m3fn)


def check_host_dtype(host_dtype) -> torch.dtype:
    """host_dtype if it is a format of the host tier (bf16, the default, or FP8 e4m3), else ValueError."""
    if host_dtype not in HOST_DTYPES:
        raise ValueError(f"K/V cache host dtype must be torch.bfloat16 or torch.float8_e4m3fn, got {host_dtype!r}")
    return host_dtype


def make_cache(num_layers: int, capacity: int, num_kv_heads: int, head_dim: int, device, *, prefill_bytes: int,
               offloaded_prefill_bytes: int, dtype=torch.bfloat16, host_dtype=torch.bfloat16):
    """The K/V cache of a generation: a KVCache when it fits on the device (device_layers), else an OffloadedKVCache
    with as many device layers as fit, its host layers in `host_dtype`.  The placement does not depend on
    host_dtype, and a KVCache ignores it.  Every buffer, host ones included, is allocated here, before the prefill."""
    check_host_dtype(host_dtype)
    row = 2 * num_kv_heads * head_dim * torch.empty((), dtype=dtype).element_size()
    n_dev = device_layers(device_free_bytes(device), capacity, num_layers, row, prefill_bytes, offloaded_prefill_bytes)
    if n_dev == num_layers:
        return KVCache(num_layers, capacity, num_kv_heads, head_dim, device, dtype)
    return OffloadedKVCache(num_layers, n_dev, capacity, num_kv_heads, head_dim, device, host_dtype=host_dtype)


class OffloadedKVCache:
    """A K/V cache whose layers [0, n_dev) are [capacity, hkv, d] device buffers, as in KVCache, and whose layers
    [n_dev, num_layers) are one pinned host buffer [capacity, 2 hkv d] bf16 each: token-major rows of K of the hkv
    heads then V of the hkv heads, the rows of the streamed layer's K|V buffer.  With host_dtype=torch.float8_e4m3fn
    a host layer is uint8 [capacity, ops.kv_fp8_row_bytes(hkv, d)] instead: the same rows quantised per head on the
    way out (ops.kv_rows_to_host_fp8) and decoded by ops.attention_decode_host_fp8.

    The first forward fills it (it may stream: the attention step declares query_chunks while the cache is empty);
    each later forward adds one token.  A multi-token forward on a filled cache (chunked prefill, a second turn) is
    refused."""

    def __init__(self, num_layers: int, n_dev: int, capacity: int, num_kv_heads: int, head_dim: int, device,
                 host_dtype=torch.bfloat16):
        if not 0 <= n_dev < num_layers:
            raise ValueError(f"OffloadedKVCache: {n_dev} device layers of {num_layers}")
        self.capacity = int(capacity)
        self.n_dev = int(n_dev)
        self.host_dtype = check_host_dtype(host_dtype)
        shape = (self.capacity, num_kv_heads, head_dim)
        self.k = [torch.empty(shape, dtype=torch.bfloat16, device=device) for _ in range(n_dev)]
        self.v = [torch.empty(shape, dtype=torch.bfloat16, device=device) for _ in range(n_dev)]
        if host_dtype == torch.float8_e4m3fn:
            self.host = [ops.pinned_fp8_rows(self.capacity, num_kv_heads, head_dim) for _ in range(num_layers - n_dev)]
        else:
            self.host = [ops.pinned_rows(self.capacity, 2 * num_kv_heads * head_dim)
                         for _ in range(num_layers - n_dev)]
        self._len = 0
        self._pending = 0

    def __len__(self) -> int:
        return self._len

    def get_seq_length(self, layer_idx: int = 0) -> int:
        return self._len

    def on_host(self, layer_idx: int) -> bool:
        return layer_idx >= self.n_dev

    def check_rows(self, rows: int) -> None:
        """Refuses a forward of `rows` new tokens that this cache cannot take (before anything is launched)."""
        if rows > 1 and self._len:
            raise NotImplementedError("a K/V cache partly in host memory takes one prompt and then one token per "
                                      "forward; a multi-token call on a filled cache (chunked prefill, a second "
                                      "turn) is not supported")

    def _rows(self, k: torch.Tensor, n: Optional[int]) -> Tuple[int, int, int]:
        """(first, end, n) of the new rows: the last n rows of k (all when None); a streamed span passes the keys up
        to its last row, of which its own are the last."""
        kr = k.shape[0]
        n = kr if n is None else n
        end = self._len + kr
        if end > self.capacity:
            raise RuntimeError(f"KV cache overflow: {end} tokens > capacity {self.capacity}")
        self._pending = kr
        return end - n, end, n

    def append(self, layer_idx: int, k: torch.Tensor, v: torch.Tensor,
               n: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor, int]:
        """A device layer: write the last `n` rows of k / v [kr, hkv, d] at rows [len + kr - n, len + kr); returns
        (K, V, len + kr) like KVCache.append."""
        r0, end, n = self._rows(k, n)
        self.k[layer_idx][r0:end].copy_(k[k.shape[0] - n :])
        self.v[layer_idx][r0:end].copy_(v[v.shape[0] - n :])
        return self.k[layer_idx], self.v[layer_idx], end

    def append_host(self, layer_idx: int, k: torch.Tensor, v: torch.Tensor,
                    n: Optional[int] = None) -> Tuple[torch.Tensor, int]:
        """A host layer: the same rows, copied device-to-host in stream order (ops.kv_rows_to_host; quantised on
        the way, ops.kv_rows_to_host_fp8, in an FP8 cache); returns (the host buffer, len + kr)."""
        r0, end, n = self._rows(k, n)
        kr = k.shape[0]
        host = self.host[layer_idx - self.n_dev]
        to_host = ops.kv_rows_to_host_fp8 if self.host_dtype == torch.float8_e4m3fn else ops.kv_rows_to_host
        to_host(k[kr - n :], v[kr - n :], host[r0:end])
        return host, end

    def decode_host(self, q: torch.Tensor, host: torch.Tensor, length: int, return_lse: bool = False):
        """One new token's attention over rows [0, length) of a host layer, in its format."""
        if self.host_dtype == torch.float8_e4m3fn:
            return ops.attention_decode_host_fp8(q, host, length, return_lse=return_lse)
        return ops.attention_decode_host(q, host, length, return_lse=return_lse)

    def commit(self) -> None:
        self._len += self._pending
        self._pending = 0

    def commit_to(self, offset: int) -> None:
        _commit_to(self, offset)

    def bytes(self) -> int:
        """Device bytes of the cache."""
        return sum(t.numel() * t.element_size() for t in self.k + self.v)

    def host_bytes(self) -> int:
        """Pinned host bytes of the cache."""
        return sum(t.numel() * t.element_size() for t in self.host)


class ContextCache:
    """The read-only K/V cache of a prefilled prompt (LongVITAForCausalLM.prefill_context): `cache` (a filled KVCache
    or OffloadedKVCache of len(cache) = P rows) and `logits`, those of the prompt's last token.  It has no append:
    questions about the prompt run in sessions of their own (session()), and the context's rows stay as they are."""

    def __init__(self, cache, logits: torch.Tensor, num_kv_heads: int, head_dim: int):
        if len(cache) == 0:
            raise ValueError("ContextCache: the cache holds no prompt")
        self.cache = cache
        self.logits = logits
        self.num_kv_heads = int(num_kv_heads)
        self.head_dim = int(head_dim)
        self.num_layers = len(cache.k) + len(getattr(cache, "host", ()))

    def __len__(self) -> int:
        return len(self.cache)

    def get_seq_length(self, layer_idx: int = 0) -> int:
        return len(self.cache)

    def session(self, max_new_rows: int) -> "ContextSession":
        """A new ContextSession with room for `max_new_rows` rows of question and answer."""
        return ContextSession(self, max_new_rows)


class ContextSession:
    """One question about a ContextCache: the context's P rows, read only, and a private device KVCache `suffix` of
    `max_new_rows` rows per layer for the question's and the answer's rows.  Used as `past_key_values`, it takes the
    cache's part: len() is P + the committed suffix rows, so positions continue at P + len(suffix), and commit /
    commit_to advance the suffix.  The attention step (hf.modeling.attention_step) attends each new row over the
    context and over the suffix, and merges the two."""

    def __init__(self, context: ContextCache, max_new_rows: int):
        if int(max_new_rows) <= 0:
            raise ValueError(f"ContextSession: max_new_rows must be positive, got {max_new_rows}")
        self.context = context
        self.prefix_len = len(context)
        self.suffix = KVCache(context.num_layers, int(max_new_rows), context.num_kv_heads, context.head_dim,
                              context.logits.device)

    def __len__(self) -> int:
        return self.prefix_len + len(self.suffix)

    def get_seq_length(self, layer_idx: int = 0) -> int:
        return len(self)

    def check_rows(self, rows: int) -> None:
        """Refuses, before anything is launched, a forward of `rows` new tokens that overflows the suffix (the error
        KVCache.append raises)."""
        end = len(self.suffix) + rows
        if end > self.suffix.capacity:
            raise RuntimeError(f"KV cache overflow: {end} tokens > capacity {self.suffix.capacity}")

    def commit(self) -> None:
        self.suffix.commit()

    def commit_to(self, offset: int) -> None:
        self.suffix.commit_to(int(offset) - self.prefix_len)
