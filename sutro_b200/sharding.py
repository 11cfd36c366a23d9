"""Row sharding across GPUs (one process per GPU, launched by torchrun).

The path is embarrassingly parallel — rows are independent and results positional
(sutro/sdk.py:406-412) — so there is no data-path collective: every rank runs the full
hot path on a contiguous block of rows with its own model replica, and the outputs are
gathered on the host (variable-length strings).  The only GPU collective is the initial
weight broadcast from rank 0 over NCCL/NVLink.
"""
from __future__ import annotations

from typing import Any, Callable, List, Optional, Sequence, Tuple


def shard_bounds(n_rows: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous balanced blocks: the first n_rows % world ranks get one extra row."""
    base, extra = divmod(n_rows, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def balanced_shards(costs: Sequence[int], world: int) -> List[List[int]]:
    """Cost-balanced assignment of rows to `world` shards (SURVEY.md §8(e): balance tokens
    rather than rows).  Rows are dealt longest-first in snake order (0..w-1, w-1..0, …), which
    keeps both the row counts (±1) and the summed cost of the shards close; every shard's
    indices come back in ascending order so results can be scattered back positionally.
    `costs` is any per-row proxy for work — the UTF-8 length of the row is what callers use."""
    shards: List[List[int]] = [[] for _ in range(world)]
    order = sorted(range(len(costs)), key=lambda i: (-int(costs[i]), i))
    for k, i in enumerate(order):
        lap, pos = divmod(k, world)
        shards[pos if lap % 2 == 0 else world - 1 - pos].append(i)
    for s in shards:
        s.sort()
    return shards


def broadcast_weights(tensors, src: int = 0) -> float:
    """NCCL broadcast of every weight tensor from `src`; returns milliseconds."""
    import time

    import torch
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return 0.0
    if tensors and tensors[0].is_cuda:
        torch.cuda.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    for t in tensors:
        dist.broadcast(t, src=src)
    if tensors and tensors[0].is_cuda:
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def infer_sharded(rows: Sequence[Any], run_shard: Callable[[Sequence[Any]], List[Any]],
                  dst: int = 0, balance: str = "rows") -> Optional[List[Any]]:
    """Run `run_shard` on this rank's share of `rows` and gather the per-row outputs, in
    the original order, on rank `dst` (other ranks get None).  `balance="rows"` gives
    contiguous blocks, `"bytes"` the cost-balanced assignment of `balanced_shards` (every
    rank computes the same assignment from the same rows, so nothing is exchanged up front).
    Works with any initialised process group (NCCL in production, gloo in the CPU tests)."""
    import torch.distributed as dist
    if balance not in ("rows", "bytes"):
        raise ValueError("balance must be 'rows' or 'bytes'")
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return list(run_shard(rows))
    world, rank = dist.get_world_size(), dist.get_rank()
    if balance == "rows":
        shards = [list(range(*shard_bounds(len(rows), world, r))) for r in range(world)]
    else:
        shards = balanced_shards([len(str(r).encode("utf-8")) if r is not None else 0
                                  for r in rows], world)
    idx = shards[rank]
    mine = list(run_shard([rows[i] for i in idx]))
    if len(mine) != len(idx):
        raise RuntimeError(f"rank {rank}: shard produced {len(mine)} outputs for {len(idx)} rows")
    parts: Optional[List[Any]] = [None] * world if rank == dst else None
    dist.gather_object(mine, parts, dst=dst)
    if rank != dst:
        return None
    out: List[Any] = [None] * len(rows)
    for ids, p in zip(shards, parts):
        for i, v in zip(ids, p):
            out[i] = v
    return out


# --------------------------------------------------------------------------- sharded frame
def snake_assignment(costs, world: int) -> List["np.ndarray"]:
    """`balanced_shards` vectorised (numpy): same shards, as sorted int64 index arrays.  At
    10^5-10^6 rows the pure-Python deal would show up next to a sub-second GPU step."""
    import numpy as np
    costs = np.asarray(costs, dtype=np.int64)
    n = len(costs)
    order = np.lexsort((np.arange(n), -costs))          # cost descending, index ascending
    k = np.arange(n)
    lap, pos = np.divmod(k, world)
    shard = np.where(lap % 2 == 0, pos, world - 1 - pos)
    return [np.sort(order[shard == r]).astype(np.int64) for r in range(world)]


def infer_frame_sharded(engine, rows=None, src: int = 0, balance: str = "bytes", **gen):
    """One frame column, all GPUs of the box — the product's multi-GPU path (one process per
    GPU under torchrun; every rank calls this, only `src` passes `rows`).

      src    rows -> Arrow blob -> HBM                                  (host -> device, once)
      all    NCCL broadcast of bytes + offsets; every rank derives the same length-balanced
             assignment (`snake_assignment` over the rows' byte lengths) and selects ITS rows
             from the resident column with a native kernel (`engine.rows_select`)
      all    `engine.run_blob_dev` on the shard: tokenise -> prefill/decode -> detokenise
      all    NCCL gather of the per-rank result columns (padded to a common size) on `src`
      src    ordered merge: the same native row-selection over the gathered parts puts
             outputs[i] next to inputs[i] (positional results, sutro/sdk.py:406-412);
             device -> host, Python strings

    Returns on `src` a dict(outputs | embeddings, stats, t_resident_s, t_results_resident_s,
    t_total_s); None on the other ranks.  With world size 1 (or no process group) the same
    code runs without the collectives.  `engine` needs `.device`, `.spec.embedding_model`,
    `rows_select(...)` and `run_blob_dev(...)` (LocalEngine; a CPU stand-in in the gloo tests);
    its `.vocab`, when it has one, decides whether `src` NFC-normalises the rows first."""
    import time

    import numpy as np
    import torch
    import torch.distributed as dist

    from .engine import blob_to_rows, normalize_rows, rows_to_blob
    if balance not in ("rows", "bytes"):
        raise ValueError("balance must be 'rows' or 'bytes'")
    multi = dist.is_initialized() and dist.get_world_size() > 1
    world = dist.get_world_size() if multi else 1
    rank = dist.get_rank() if multi else 0
    dev = engine.device
    emb_mode = bool(engine.spec.embedding_model)
    is_cuda = dev.type == "cuda"

    def sync():
        if is_cuda:
            torch.cuda.synchronize(dev)

    t0 = time.perf_counter()
    # ---- src: the column becomes resident in HBM ---------------------------------------
    if rank == src:
        if rows is None:
            raise ValueError("the source rank must pass the rows")
        data, off = rows_to_blob(normalize_rows(rows, getattr(engine, "vocab", None)))
        n_rows, n_bytes = len(off) - 1, int(off[-1])
        hdr = torch.tensor([n_rows, n_bytes], dtype=torch.int64, device=dev)
        d_text = torch.from_numpy(np.ascontiguousarray(data)).to(dev) if n_bytes else \
            torch.zeros(1, dtype=torch.uint8, device=dev)
        d_off = torch.from_numpy(np.ascontiguousarray(off, dtype=np.int64)).to(dev)
        h2d = int(data.nbytes + off.nbytes)
    else:
        hdr = torch.zeros(2, dtype=torch.int64, device=dev)
        h2d = 0
    sync()
    t_res = time.perf_counter()
    ev = None
    if is_cuda:    # device time of "column resident -> ordered results resident" on this rank
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    if multi:
        dist.broadcast(hdr, src=src)
        n_rows, n_bytes = (int(x) for x in hdr.cpu())
        if rank != src:
            d_text = torch.empty(max(n_bytes, 1), dtype=torch.uint8, device=dev)
            d_off = torch.empty(n_rows + 1, dtype=torch.int64, device=dev)
        dist.broadcast(d_text, src=src)
        dist.broadcast(d_off, src=src)
    if n_rows == 0:
        return dict(outputs=[], embeddings=None, stats={"n_rows": 0}, t_total_s=0.0) \
            if rank == src else None

    # ---- every rank: same assignment, own rows ------------------------------------------
    if world > 1:
        off_h = off if rank == src else d_off.cpu().numpy()
        lens = np.diff(off_h)
        if balance == "bytes":
            shards = snake_assignment(lens, world)
        else:
            shards = [np.arange(*shard_bounds(n_rows, world, r), dtype=np.int64)
                      for r in range(world)]
        idx = shards[rank]
        m = len(idx)
        d_idx = torch.from_numpy(idx).to(dev)
        d_soff, d_sbytes = engine.rows_select(d_text, d_off, n_rows, 0, d_idx, n_bytes)
        s_bytes = int(d_soff[-1].item()) if m else 0
        r = engine.run_blob_dev(d_sbytes, d_soff, m, s_bytes, row_ids=idx, **gen) if m else None
    else:
        shards, idx, m = None, None, n_rows
        r = engine.run_blob_dev(d_text, d_off, n_rows, n_bytes, **gen)

    # ---- gather on src, ordered merge ------------------------------------------------------
    out: dict = {}
    if world == 1:
        if ev:
            ev[1].record()
        sync()
        t_out = time.perf_counter()
        if emb_mode:
            out["embeddings"] = r["d_emb"].cpu().numpy()
            d2h = out["embeddings"].nbytes
        else:
            b, boff = r["d_bytes"].cpu().numpy(), r["d_boff"].cpu().numpy()
            out["outputs"] = blob_to_rows(b, boff)
            d2h = b.nbytes + boff.nbytes
        stats = [r["stats"]]
    else:
        max_m = max(len(s) for s in shards)
        if emb_mode:
            d = engine.spec.d_model
            part = torch.zeros(max_m, d, dtype=torch.float32, device=dev)
            if m:
                part[:m] = r["d_emb"]
            parts = [torch.empty_like(part) for _ in range(world)] if rank == src else None
            dist.gather(part, parts, dst=src)
        else:
            my_b = int(r["d_boff"][-1].item()) if m else 0
            sizes = torch.tensor([my_b], dtype=torch.int64, device=dev)
            all_sizes = [torch.zeros_like(sizes) for _ in range(world)]
            dist.all_gather(all_sizes, sizes)
            max_b = max(1, max(int(s.item()) for s in all_sizes))
            pb = torch.zeros(max_b, dtype=torch.uint8, device=dev)
            po = torch.zeros(max_m + 1, dtype=torch.int64, device=dev)
            if m:
                pb[:my_b] = r["d_bytes"][:my_b]
                po[:m + 1] = r["d_boff"]
                po[m + 1:] = my_b
            gb = go = None
            if rank == src:   # the parts land side by side: one batch of equally strided columns
                bytes_all = torch.empty(world * max_b, dtype=torch.uint8, device=dev)
                off_all = torch.empty(world * (max_m + 1), dtype=torch.int64, device=dev)
                gb, go = list(bytes_all.split(max_b)), list(off_all.split(max_m + 1))
            dist.gather(pb, gb, dst=src)
            dist.gather(po, go, dst=src)
        my_stats = None if r is None else {k: v for k, v in r["stats"].items()}
        stats = [None] * world if rank == src else None
        dist.gather_object(my_stats, stats, dst=src)
        if rank != src:
            return None
        if emb_mode:
            if ev:
                ev[1].record()
            sync()
            t_out = time.perf_counter()
            emb = np.empty((n_rows, engine.spec.d_model), dtype=np.float32)
            for ids, p in zip(shards, parts):
                emb[ids] = p[:len(ids)].cpu().numpy()
            out["embeddings"] = emb
            d2h = emb.nbytes
        else:
            # global row i sits at (part, local) -> row part*max_m + local of the batch of parts
            sel = np.empty(n_rows, dtype=np.int64)
            for p, ids in enumerate(shards):
                sel[ids] = p * max_m + np.arange(len(ids), dtype=np.int64)
            d_sel = torch.from_numpy(sel).to(dev)
            d_ooff, d_obytes = engine.rows_select(bytes_all, off_all, max_m, max_b, d_sel,
                                                  int(bytes_all.numel()))
            if ev:
                ev[1].record()
            sync()
            t_out = time.perf_counter()
            boff = d_ooff.cpu().numpy()
            b = d_obytes[:int(boff[-1])].cpu().numpy()
            out["outputs"] = blob_to_rows(b, boff)
            d2h = b.nbytes + boff.nbytes
    t_end = time.perf_counter()
    agg = {"n_gpus": world, "n_rows": n_rows, "h2d_bytes": h2d, "d2h_bytes": int(d2h),
           "per_gpu": stats,
           "t_device_ms": ev[0].elapsed_time(ev[1]) if ev else 1e3 * (t_out - t_res)}
    for k in ("input_tokens", "output_tokens", "decode_tokens", "prefill_tokens", "rows_done",
              "rows_truncated", "prefill_steps", "decode_steps"):
        agg[k] = sum(int(s.get(k, 0)) for s in stats if s)
    out.update(stats=agg, t_resident_s=t_res - t0, t_results_resident_s=t_out - t0,
               t_total_s=t_end - t0)
    return out
