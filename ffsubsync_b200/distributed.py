"""Multi-GPU plumbing: one process per GPU, pairs block-sharded over ranks, NCCL (over NVLink /
NVSwitch) only for the final exchange of per-pair results (SURVEY.md section 8e).

The path shards without any data-path collective: pairs are independent and all K ratio
candidates of a pair stay on one GPU, so the max over ratios (b2_reduce_ratios) is local.  The
only communication is the gather of ``(score, offset, ratio index)`` - 16 bytes per pair - to
rank 0 (primary mode), or an all-gather of per-candidate results when the K candidates of a
few pairs are spread over ranks (secondary mode, B < world size).  Messages are bytes to KB:
latency-bound, one collective per batch.

The same functions run on the ``gloo`` backend with CPU tensors (tests, world_size 2).
"""
import os
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.distributed as dist


def init_from_env(backend: Optional[str] = None) -> Tuple[int, int, int]:
    """(rank, world_size, local_rank) from the torchrun environment; initialises the default
    process group when WORLD_SIZE > 1."""
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29531")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local_rank)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local_rank


def _parse_cpulist(text: str) -> set:
    cpus = set()
    for part in text.strip().split(","):
        if not part:
            continue
        lo, _, hi = part.partition("-")
        cpus.update(range(int(lo), int(hi or lo) + 1))
    return cpus


def gpu_numa_node(device_index: int) -> Tuple[int, str]:
    """(NUMA node of the GPU's PCIe root, PCI bus id) from sysfs; node -1 when unknown."""
    bus = None
    try:
        p = torch.cuda.get_device_properties(device_index)
        bus = "%04x:%02x:%02x.0" % (p.pci_domain_id, p.pci_bus_id, p.pci_device_id)
    except Exception:
        try:
            import pynvml
            pynvml.nvmlInit()
            info = pynvml.nvmlDeviceGetPciInfo(pynvml.nvmlDeviceGetHandleByIndex(device_index))
            raw = info.busId.decode() if isinstance(info.busId, bytes) else info.busId
            bus = raw.lower()[-12:]
        except Exception:
            return -1, ""
    try:
        with open("/sys/bus/pci/devices/%s/numa_node" % bus) as fh:
            return int(fh.read().strip()), bus
    except (OSError, ValueError):
        return -1, bus


def bind_to_gpu_numa(local_rank: int) -> dict:
    """Pin this process to the CPU cores of its GPU's NUMA node (call before allocating pinned host
    buffers: first touch then places them on that node, so H2D copies do not cross the socket
    interconnect).  Returns what was done, for the bench record; never raises."""
    info = {"node": -1, "bound": False}
    try:
        node, bus = gpu_numa_node(local_rank)
        info.update(node=node, pci=bus)
        if node < 0:
            return info
        with open("/sys/devices/system/node/node%d/cpulist" % node) as fh:
            cpus = _parse_cpulist(fh.read())
        allowed = os.sched_getaffinity(0) & cpus
        if allowed:
            os.sched_setaffinity(0, allowed)
            info.update(bound=True, cpus=len(allowed))
    except Exception as e:  # containers may hide sysfs or forbid sched_setaffinity
        info["error"] = str(e)
    return info


def shard_pairs(n_pairs: int, rank: int, world: int) -> Tuple[int, int]:
    """Block sharding: rank g owns pairs [g*B/G, (g+1)*B/G)."""
    return (rank * n_pairs) // world, ((rank + 1) * n_pairs) // world


def shard_candidates(n_candidates: int, rank: int, world: int) -> List[int]:
    """Secondary mode: candidate k of every pair goes to rank k % world (keeps list order inside
    a rank, so "first in list wins" can be restored after the all-gather)."""
    return list(range(rank, n_candidates, world))


def shard_videos(track_video, rank: int, world: int) -> Tuple[int, int, int, int]:
    """Block sharding of videos with several subtitle tracks (track_video: non-decreasing video index of
    each track, as for BatchSynchronizer.sync_device_tracks).  Rank g owns the videos [v0, v1) and their
    tracks [t0, t1); a video's tracks never straddle two ranks, and the rank boundaries are the first
    videos whose tracks start at or after track g*T/G, so ranks hold about equal numbers of tracks.
    The videos are those up to the last one with tracks (V = track_video[-1] + 1); one without tracks
    goes with the previous video that has tracks.  Returns (v0, v1, t0, t1)."""
    track_video = np.asarray(track_video, dtype=np.int64)
    T = len(track_video)
    V = int(track_video[-1]) + 1 if T else 0

    def cut(g):
        if g >= world:
            return V, T
        t = (g * T) // world
        while 0 < t < T and track_video[t] == track_video[t - 1]:   # move up to the start of the next video
            t += 1
        return (int(track_video[t]) if t < T else V), t

    (v0, t0), (v1, t1) = cut(rank), cut(rank + 1)
    return (0 if rank == 0 else v0), v1, t0, t1


def _gather_blocks(local: torch.Tensor, counts: List[Tuple[int, int]], rank: int, world: int, dst: Optional[int],
                   group) -> Optional[torch.Tensor]:
    """Rank r holds rows [lo_r, hi_r) of the result: pad every block to the largest, one
    all_gather_into_tensor, concatenate in rank order on ``dst`` (every rank when dst is None)."""
    width = max(max(hi - lo for lo, hi in counts), 1)
    padded = torch.zeros((width,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    padded[: local.shape[0]] = local
    out = torch.empty((world * width,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, padded, group=group)
    if dst is not None and rank != dst:
        return None
    out = out.view((world, width) + tuple(local.shape[1:]))
    return torch.cat([out[r, : hi - lo] for r, (lo, hi) in enumerate(counts)], dim=0)


def _gather_any(local, counts, rank, world, dst, group):
    """A tensor, or a dict of per-row tensors such as BatchSynchronizer.sync_device's output (best_*, and
    gss_ratio with the golden-section search): every entry is gathered the same way, one collective each."""
    if not isinstance(local, dict):
        return _gather_blocks(local, counts, rank, world, dst, group)
    out = {k: _gather_blocks(v, counts, rank, world, dst, group) for k, v in local.items()}
    return None if dst is not None and rank != dst else out


def gather_pair_results(local, n_pairs: int, rank: int, world: int, dst: int = 0, group=None):
    """local: [n_local, C] results of this rank's block of pairs (any dtype, same on all ranks), or a dict
    of such tensors (e.g. sync_device's output, which carries gss_ratio with the golden-section search).
    Returns [n_pairs, C] (or the dict of them) in global pair order on ``dst`` (None elsewhere).  One
    collective per tensor."""
    if world == 1:
        return local
    return _gather_any(local, [shard_pairs(n_pairs, r, world) for r in range(world)], rank, world, dst, group)


def gather_track_results(local, track_video, rank: int, world: int, dst: Optional[int] = 0, group=None):
    """local: [t1 - t0, C] results of the tracks shard_videos() gave this rank (per-rank counts differ), or a
    dict of such tensors (e.g. sync_device_tracks' output, which carries gss_ratio with the golden-section
    search).  Returns [T, C] (or the dict of them) in global track order on ``dst`` (on every rank when dst is
    None, None elsewhere).  One collective per tensor."""
    if world == 1:
        return local
    counts = [shard_videos(track_video, r, world)[2:] for r in range(world)]
    return _gather_any(local, counts, rank, world, dst, group)


def allgather_candidate_results(local: torch.Tensor, n_candidates: int, rank: int, world: int,
                                group=None) -> torch.Tensor:
    """Secondary mode.  local: [B, K_local, C] for the candidates shard_candidates() gave this
    rank.  Returns [B, K, C] with candidates back in list order on every rank, ready for
    b2_reduce_ratios (which then applies the |offset| filter and first-wins tie rule)."""
    if world == 1:
        return local
    B, C = local.shape[0], local.shape[2]
    width = (n_candidates + world - 1) // world
    padded = torch.zeros((B, width, C), dtype=local.dtype, device=local.device)
    padded[:, : local.shape[1]] = local
    out = torch.empty((world, B, width, C), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out.view(world * B, width, C), padded, group=group)
    full = torch.empty((B, n_candidates, C), dtype=local.dtype, device=local.device)
    for r in range(world):
        ks = shard_candidates(n_candidates, r, world)
        if ks:
            full[:, ks] = out[r, :, : len(ks)]
    return full


def max_over_ranks(value: float, device=None) -> float:
    """Timing helper: the slowest rank defines the step time."""
    if not dist.is_initialized():
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
