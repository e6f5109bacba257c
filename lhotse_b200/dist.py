"""
Multi-GPU plumbing: one process per GPU, cuts sharded across ranks, no data-path collective.

The path is embarrassingly parallel (cuts are independent), so the only communication is
  * a broadcast of the constant-table blob from rank 0 at start-up (every rank then runs on
    bit-identical window / mel / DCT tables), and
  * reductions of counters / elapsed time for reporting.
Sharding is the reference's own job split: rank r of W takes cuts r, r+W, ...
(`LazySlicer(k=r, n=W)`, lhotse/cut/set.py:2158-2160; sampler-level equivalent
lhotse/dataset/sampling/base.py:143-164).
"""
from __future__ import annotations

import os
from typing import Iterable, Iterator, List, Optional, Sequence, Tuple, TypeVar

import numpy as np
import torch
import torch.distributed as dist

from .plan import FeaturePlan

T = TypeVar("T")


def env_rank_world() -> Tuple[int, int, int]:
    return (int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0)))


def init_distributed(backend: Optional[str] = None) -> Tuple[int, int, int]:
    """Initialises torch.distributed from the torchrun environment (no-op for world size 1).  Returns (rank, world, device index).

    More local ranks than GPUs is allowed for the host-bound jobs (the CutSet-level store spends > 95 % of its wall clock in
    per-cut Python — manifests, sampler — so several processes per GPU multiply its throughput): local rank r then uses GPU
    r mod #GPUs, and the job-level collectives (table broadcast, barriers, timing reductions) run over gloo, because NCCL
    refuses two ranks on one device.  `bench.py` itself always runs one rank per GPU."""
    rank, world, local = env_rank_world()
    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    oversubscribed = ngpu > 0 and int(os.environ.get("LOCAL_WORLD_SIZE", world)) > ngpu
    if ngpu > 0:
        local = local % ngpu
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if ngpu > 0 and not oversubscribed else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        kw = {}
        if backend == "nccl":
            torch.cuda.set_device(local)
            kw["device_id"] = torch.device("cuda", local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world, **kw)
    return rank, world, local


def gpu_numa_node(device_index: int) -> Optional[int]:
    """NUMA node of a CUDA device (sysfs `numa_node` of its PCI function), or None when the platform does not say."""
    try:
        pr = torch.cuda.get_device_properties(device_index)
        path = f"/sys/bus/pci/devices/{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0/numa_node"
        with open(path) as f:
            node = int(f.read().strip())
        return node if node >= 0 else None
    except (OSError, ValueError, AttributeError, RuntimeError):
        return None


def _parse_cpulist(text: str) -> List[int]:
    cpus: List[int] = []
    for part in text.strip().split(","):
        if not part:
            continue
        lo, _, hi = part.partition("-")
        cpus.extend(range(int(lo), int(hi or lo) + 1))
    return cpus


def bind_host_to_gpu_numa(device_index: int) -> Optional[int]:
    """Pins this process to the CPUs of the NUMA node its GPU hangs off, so that the pinned staging buffers it allocates
    next (first touch) and the threads that fill them are local to the GPU's PCIe root.  One process per GPU is the
    deployment model (torchrun), so this is a per-rank decision.  On a two-socket box with 8 GPUs the host-to-host rate is
    bound by host memory traffic, and remote (cross-socket) pinned buffers halve it.  Returns the node, or None when
    nothing was changed (single node, no permission, unknown topology).  `B200FEAT_NO_NUMA_BIND=1` disables it."""
    if os.environ.get("B200FEAT_NO_NUMA_BIND") == "1" or not hasattr(os, "sched_setaffinity"):
        return None
    node = gpu_numa_node(device_index)
    if node is None:
        return None
    try:
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = set(_parse_cpulist(f.read()))
        allowed = os.sched_getaffinity(0)
        target = cpus & allowed
        if not target or target == allowed:
            return None
        os.sched_setaffinity(0, target)
        return node
    except (OSError, ValueError):
        return None


def shard_slice(items: Sequence[T], rank: int, world: int) -> List[T]:
    """rank::world striding — identical to LazySlicer(k=rank, n=world)."""
    return list(items[rank::world])


def shard_iter(items: Iterable[T], rank: int, world: int) -> Iterator[T]:
    for i, it in enumerate(items):
        if i % world == rank:
            yield it


def unshard(per_rank: Sequence[Sequence[T]]) -> List[T]:
    """Inverse of shard_slice over all ranks (the order `combine` restores)."""
    world = len(per_rank)
    total = sum(len(p) for p in per_rank)
    out: List[Optional[T]] = [None] * total
    for r, part in enumerate(per_rank):
        out[r::world] = list(part)
    return out  # type: ignore


def _comm_device() -> torch.device:
    if dist.is_initialized() and dist.get_backend() == "nccl":
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def broadcast_plan_tables(plan: FeaturePlan, src: int = 0) -> FeaturePlan:
    """Every rank ends up with rank `src`'s float32 tables, bit for bit (~90 KB over NCCL/NVLink)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return plan
    blob = torch.from_numpy(plan.tables_blob()).to(_comm_device())
    dist.broadcast(blob, src=src)
    plan.load_tables_blob(blob.cpu().numpy())
    return plan


def all_reduce_stats(values: Sequence[float], op: str = "sum") -> List[float]:
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return list(values)
    t = torch.tensor(list(values), dtype=torch.float64, device=_comm_device())
    dist.all_reduce(t, op={"sum": dist.ReduceOp.SUM, "max": dist.ReduceOp.MAX, "min": dist.ReduceOp.MIN}[op])
    return t.cpu().tolist()


def barrier():
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()


def compute_and_store_features_sharded(cuts, extractor, storage_path, rank: Optional[int] = None,
                                       world: Optional[int] = None, manifest_name: str = "cuts", fused: bool = False,
                                       **kwargs):
    """§8e partitioning through lhotse's own batch caller: rank r of W extracts cuts r::W with
    ``CutSet.compute_and_store_features_batch`` (lhotse/cut/set.py:2197) into ``storage_path/feats-{r}``
    and writes ``storage_path/{manifest_name}-{r}.jsonl.gz`` — the layout the reference's ``num_jobs`` split
    produces (set.py:2158-2195), so lhotse's resume logic (``overwrite=False``) and ``combine`` apply per shard.
    With ``fused=True`` the shard goes through ``lhotse_b200.storage.compute_and_store_features_fused`` instead (one
    packed extraction, one D2H copy, one append to ``storage_path/feats-{r}.b200feat`` per batch; same manifests).
    Returns this rank's CutSet with features attached.  Needs lhotse."""
    from pathlib import Path

    from lhotse import CutSet

    if rank is None or world is None:
        r, w, _ = env_rank_world()
        rank = r if rank is None else rank
        world = w if world is None else world
    storage_path = Path(storage_path)
    storage_path.mkdir(parents=True, exist_ok=True)
    mine = CutSet.from_cuts(shard_iter(cuts, rank, world))
    if fused:
        from .storage import compute_and_store_features_fused

        allowed = {k: v for k, v in kwargs.items() if k in ("batch_duration", "num_workers", "overwrite", "pcm16_fast_path",
                                                            "reverb", "generated_rir", "wpe")}
        return compute_and_store_features_fused(mine, extractor, storage_path / f"feats-{rank}",
                                                manifest_path=storage_path / f"{manifest_name}-{rank}.jsonl.gz", **allowed)
    return mine.compute_and_store_features_batch(
        extractor=extractor,
        storage_path=storage_path / f"feats-{rank}",
        manifest_path=storage_path / f"{manifest_name}-{rank}.jsonl.gz",
        **kwargs,
    )


def combine_shards(storage_path, world: int, manifest_name: str = "cuts"):
    """Rank-0 epilogue: one lazy CutSet over the per-rank manifests, in the original cut order."""
    from pathlib import Path

    from lhotse import CutSet, load_manifest_lazy

    shards = [list(load_manifest_lazy(Path(storage_path) / f"{manifest_name}-{r}.jsonl.gz")) for r in range(world)]
    return CutSet.from_cuts(unshard(shards))
