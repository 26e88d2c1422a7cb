"""Row sharding across GPUs: one process per GPU, W/b replicated, labels exchanged once.

The reference has no distributed path (scale-out = independent Flyte pods, ``unionml:unionml/model.py:1160-1226``);
rows are independent, so rank r scores a contiguous row block ``[r*N/G, (r+1)*N/G)`` and every rank ends up with the
full label vector (SURVEY.md 8e).  Exchange back-ends:

* ``nccl``  - ``torch.distributed.all_gather_into_tensor`` of the label vector after the kernel;
* ``fused`` - the scoring kernel's epilogue stores each label into every peer's vector over NVLink
  (``uml_linear_predict_peers`` / ``uml_mlp_predict_peers``; peer pointers or the NVLS multicast alias from
  ``torch.distributed._symmetric_memory``), followed by one symmetric-memory barrier.  No separate collective kernel,
  no extra pass over the labels;
* ``push``  - the kernel stores its labels locally and a thin copy kernel pushes the slice to the peers; with
  ``pipeline=k`` the shard is scored as k sub-batches and the push of sub-batch j runs on a side stream under the
  scoring kernel of sub-batch j+1, so back-pressure from the fabric never stalls the scoring warps.

Stream contract: ``predict_sharded`` runs the engine on torch's *current* stream for the duration of the call, so the
collective / barrier that follows the kernels is ordered after them whatever stream the engine was created with.

The host-side logic (``shard_bounds``, ``gather_labels``) is backend-agnostic and covered by world_size-2 ``gloo`` tests.
"""
import contextlib
from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n_rows: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous block ``[lo, hi)`` of rank ``rank``; the first ``n_rows % world`` ranks hold one extra row."""
    if not (0 <= rank < world):
        raise ValueError(f"rank {rank} outside world of {world}")
    base, extra = divmod(n_rows, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_counts(n_rows: int, world: int) -> List[int]:
    return [shard_bounds(n_rows, r, world)[1] - shard_bounds(n_rows, r, world)[0] for r in range(world)]


def gather_labels(local: torch.Tensor, counts: Sequence[int], group=None) -> torch.Tensor:
    """All-gather per-rank label vectors (possibly ragged) into the full vector, on whatever backend ``group`` uses."""
    world = dist.get_world_size(group)
    if len(counts) != world:
        raise ValueError("counts must have one entry per rank")
    if local.numel() != counts[dist.get_rank(group)]:
        raise ValueError("local label vector does not match this rank's shard size")
    if len(set(counts)) == 1:
        out = torch.empty(sum(counts), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    width = max(counts)
    padded = torch.zeros(width, dtype=local.dtype, device=local.device)
    padded[: local.numel()] = local
    buf = torch.empty(world * width, dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(buf, padded, group=group)
    return torch.cat([buf[r * width : r * width + counts[r]] for r in range(world)])


class PeerLabelExchange:
    """A full-length label vector (int32, or uint8 on the wire) in symmetric memory on every rank + peer pointers."""

    def __init__(self, total_rows: int, device: torch.device, group=None, dtype: torch.dtype = torch.int32,
                 multicast: bool = True, push: bool = False, pipeline: int = 1):
        import torch.distributed._symmetric_memory as symm_mem

        if dtype not in (torch.int32, torch.uint8):
            raise ValueError("label vectors are int32 or uint8 (byte labels need n_classes <= 256)")
        self.group = group if group is not None else dist.group.WORLD
        self.label_bytes = 1 if dtype == torch.uint8 else 4
        self.labels = symm_mem.empty(total_rows, dtype=dtype, device=device)
        self.handle = symm_mem.rendezvous(self.labels, self.group)
        self.rank = self.handle.rank
        self.world = self.handle.world_size
        self.push = push  # two-step variant: kernel stores locally, a thin copy kernel pushes the slice to the peers
        self.pipeline = max(1, int(pipeline)) if push else 1
        self.side_stream = torch.cuda.Stream(device=device) if self.pipeline > 1 else None
        self._sub_batches = {}
        ptrs = list(self.handle.buffer_ptrs)
        self.own_ptr = ptrs[self.rank]
        mc = int(getattr(self.handle, "multicast_ptr", 0) or 0) if multicast else 0
        self.multicast = mc != 0
        if self.multicast:
            # NVLS: one store to the multicast address is replicated by the switch into every rank's vector (own
            # included), so the kernel issues a single store per tile however many GPUs take part
            self.peer_ptrs = [mc]
        else:
            # own pointer first: the kernel treats entry 0 as its local label vector
            self.peer_ptrs = [ptrs[self.rank]] + [p for r, p in enumerate(ptrs) if r != self.rank]

    def barrier(self) -> None:
        """All ranks' stores have landed everywhere (device-side barrier on the current stream)."""
        self.handle.barrier()

    def sub_batches(self, engine, batch, k: int):
        """``k`` row slices of a resident batch (tile-aligned boundaries), wrapped once and cached."""
        key = (id(batch), k)
        hit = self._sub_batches.get(key)
        if hit is None:
            step = (batch.n_rows + k - 1) // k
            step = (step + 511) // 512 * 512  # whole tiles, and 4-byte aligned byte-label words
            hit = []
            for lo in range(0, batch.n_rows, step):
                n = min(step, batch.n_rows - lo)
                hit.append((lo, n, engine.wrap_device(batch.device_ptr + lo * batch.ld * 4, n, batch.n_features, batch.ld,
                                                      keepalive=batch)))
            self._sub_batches = {key: hit}  # one resident batch at a time
        return hit


@contextlib.contextmanager
def _engine_on_current_stream(engine, device_index):
    """Launch the engine's kernels on torch's current stream for the duration (restored afterwards)."""
    set_stream = getattr(engine, "set_stream", None)
    if set_stream is None or not torch.cuda.is_available():
        yield
        return
    prev = getattr(engine, "stream", None)
    cur = torch.cuda.current_stream(device_index).cuda_stream
    if cur == 0:
        # the legacy default stream has handle 0, which the ABI reads as "the engine's own stream": order the two by
        # draining the engine stream before the collective instead
        try:
            yield
        finally:
            engine.synchronize()
        return
    set_stream(cur)
    try:
        yield
    finally:
        set_stream(prev)


def _predict_peers(engine, model, batch, ptrs, row_offset, exact, label_bytes):
    """Dispatch on the model kind: linear classifier or 2-layer MLP, same fused-exchange contract."""
    if type(model).__name__ == "MlpModel":
        return engine.predict_mlp_peers(model, batch, ptrs, row_offset, exact=exact, label_bytes=label_bytes)
    return engine.predict_peers(model, batch, ptrs, row_offset, exact=exact, label_bytes=label_bytes)


def predict_sharded(engine, model, batch, *, row_offset: int, counts: Sequence[int], exact: bool = True,
                    exchange: Optional[PeerLabelExchange] = None, labels_all: Optional[torch.Tensor] = None,
                    group=None) -> torch.Tensor:
    """Score this rank's resident shard and return the full label vector (device tensor, identical on all ranks).

    The engine is driven on torch's current stream for the duration of the call, so the exchange is ordered after the
    kernels (a default ``Engine`` otherwise launches on its own non-blocking stream)."""
    rank = dist.get_rank(group)
    dev_index = getattr(engine, "device", 0)
    with _engine_on_current_stream(engine, dev_index):
        if exchange is not None and exchange.push:
            lb = exchange.label_bytes
            remote = exchange.peer_ptrs if exchange.multicast else exchange.peer_ptrs[1:]
            if exchange.pipeline > 1 and remote:
                main = torch.cuda.current_stream(dev_index)
                side = exchange.side_stream
                side.wait_stream(main)
                for lo, n, sub in exchange.sub_batches(engine, batch, exchange.pipeline):
                    _predict_peers(engine, model, sub, [exchange.own_ptr], row_offset + lo, exact, lb)
                    ev = torch.cuda.Event()
                    ev.record(main)
                    side.wait_event(ev)
                    off = (row_offset + lo) * lb
                    engine.set_stream(side.cuda_stream)
                    engine.push_labels(exchange.own_ptr + off, [p + off for p in remote], n * lb)
                    engine.set_stream(main.cuda_stream)
                main.wait_stream(side)
            else:
                _predict_peers(engine, model, batch, [exchange.own_ptr], row_offset, exact, lb)
                off = row_offset * lb
                if remote:
                    engine.push_labels(exchange.own_ptr + off, [p + off for p in remote], counts[rank] * lb)
            exchange.barrier()
            return exchange.labels
        if exchange is not None:
            _predict_peers(engine, model, batch, exchange.peer_ptrs, row_offset, exact, exchange.label_bytes)
            exchange.barrier()
            return exchange.labels
        if labels_all is None:
            labels_all = torch.empty(sum(counts), dtype=torch.int32, device=torch.device("cuda", engine.device))
        local = labels_all[row_offset : row_offset + counts[rank]]
        if type(model).__name__ == "MlpModel":
            engine.predict_mlp(model, batch, exact=exact, out_device_ptr=local.data_ptr(), want_stats=False)
        else:
            engine.predict(model, batch, exact=exact, out_device_ptr=local.data_ptr(), want_stats=False)
    if len(set(counts)) == 1:
        dist.all_gather_into_tensor(labels_all, local, group=group)
        return labels_all
    return gather_labels(local.clone(), counts, group)
