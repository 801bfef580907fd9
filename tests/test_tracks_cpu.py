"""CPU suite for syncing several subtitle tracks per video: the b2_sync_tracks entry point is exported
and refuses to run without a GPU, video sharding over ranks, and the per-track result gather over a
world_size-2 gloo group."""
import ctypes
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from conftest import ROOT


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()
    return ge


def test_sync_tracks_is_exported(built):
    from ffsubsync_b200 import _native
    assert "b2_sync_tracks" in _native.EXPORTS
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), "b2_sync_tracks")
    # a handle-less call is refused before anything is read
    assert _native.load().b2_sync_tracks(None, None, None, 0, None, 0, 16000, 100, 0.0, 0, -1, -1, None, None,
                                         None, None, None, 1, 0.0, 0, None, None, None, None, None, 0) == -1


def test_sync_tracks_raises_without_gpu(built):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from ffsubsync_b200 import _native
    with pytest.raises(_native.NativeError):
        h = _native.get_handle()
        h.sync_tracks(np.zeros(1600, np.int16), [0, 1600], [0], 16000, 100, 0.0, 100000, -1, -1,
                      [1.0], [2.0], None, [0, 1], [1.0], 0.0, 100)


def _check_shards(track_video, world):
    from ffsubsync_b200.distributed import shard_videos
    track_video = np.asarray(track_video)
    T = len(track_video)
    V = int(track_video[-1]) + 1 if T else 0
    shards = [shard_videos(track_video, r, world) for r in range(world)]
    # videos and tracks both partitioned, in order
    assert shards[0][0] == 0 and shards[-1][1] == V
    assert shards[0][2] == 0 and shards[-1][3] == T
    for a, b in zip(shards, shards[1:]):
        assert a[1] == b[0] and a[3] == b[2]
    for v0, v1, t0, t1 in shards:
        # a rank's tracks are exactly the tracks of its videos: no video is split
        assert np.all((track_video[t0:t1] >= v0) & (track_video[t0:t1] < v1))
        assert not np.any((track_video[:t0] >= v0) & (track_video[:t0] < v1))
        assert not np.any((track_video[t1:] >= v0) & (track_video[t1:] < v1))
    return shards


def test_shard_videos_covers_everything_without_splitting_videos():
    rng = np.random.RandomState(3)
    for world in (1, 2, 3, 4, 8):
        _check_shards([], world)
        _check_shards([0], world)
        _check_shards(np.arange(17), world)
        for _ in range(20):
            counts = rng.randint(0, 6, rng.randint(1, 40))
            counts[-1] = max(counts[-1], 1)   # the last video defines V
            _check_shards(np.repeat(np.arange(len(counts)), counts), world)


def test_shard_videos_balances_skewed_track_counts():
    # one video with many tracks among many single-track videos: each rank's track count lies within
    # the largest video of the even share
    counts = np.array([1] * 30 + [12] + [1] * 30 + [3] * 10)
    track_video = np.repeat(np.arange(len(counts)), counts)
    T = len(track_video)
    for world in (2, 4, 8):
        shards = _check_shards(track_video, world)
        for v0, v1, t0, t1 in shards:
            assert abs((t1 - t0) - T / world) <= counts.max()
    # identity map: the same blocks as shard_pairs
    from ffsubsync_b200.distributed import shard_pairs, shard_videos
    for world in (2, 4):
        for r in range(world):
            v0, v1, t0, t1 = shard_videos(np.arange(13), r, world)
            assert (v0, v1) == (t0, t1) == shard_pairs(13, r, world)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from ffsubsync_b200 import distributed as D
    r, w, _ = D.init_from_env("gloo")
    assert (r, w) == (rank, world)
    # 5 videos with 5, 0, 2, 3, 2 tracks: video 2 straddles track 6, so the ranks hold 7 and 5 tracks
    track_video = np.repeat(np.arange(5), [5, 0, 2, 3, 2])
    v0, v1, t0, t1 = D.shard_videos(track_video, rank, world)
    local = torch.tensor([[1000.0 + t, -t, track_video[t]] for t in range(t0, t1)], dtype=torch.float64)
    want = torch.tensor([[1000.0 + t, -t, track_video[t]] for t in range(len(track_video))], dtype=torch.float64)
    got = D.gather_track_results(local, track_video, rank, world)
    if rank == 0:
        assert torch.equal(got, want)
    else:
        assert got is None
    assert torch.equal(D.gather_track_results(local, track_video, rank, world, dst=None), want)
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()
    q.put((rank, (t1 - t0, "ok")))


def test_gather_track_results_gloo_world_size_2():
    world = 2
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    got = sorted(q.get(timeout=5) for _ in range(world))
    assert [r for r, _ in got] == [0, 1] and all(res[1] == "ok" for _, res in got)
    assert got[0][1][0] != got[1][1][0]   # unequal per-rank counts were exercised
