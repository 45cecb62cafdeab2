"""The file agreement of a sharded --partition-tag run (agree_file_slices, through mkh_agree_file_slices), without a GPU: every
rank learns the union of the file names, its offset in each file and each file's total size, for 1 to 8 ranks with random
name -> size maps (names on one rank only, zero-byte names, ranks with no files). The ranks run as threads over an in-process
sum that records every call's length, and once as processes over gloo through modkit_b200.torch_allreduce."""
import os
import random
import socket
import threading

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import modkit_b200


class ThreadSum:
    """A u64 sum over `world` threads; records the length of every call of every rank."""

    def __init__(self, world):
        self.world = world
        self.bar = threading.Barrier(world)
        self.bufs = [None] * world
        self.calls = [[] for _ in range(world)]

    def for_rank(self, rank):
        def fn(buf, n, _user):
            try:
                a = np.ctypeslib.as_array(buf, shape=(n,))
                self.calls[rank].append(n)
                self.bufs[rank] = a.copy()
                self.bar.wait(timeout=60)
                if len({len(b) for b in self.bufs}) != 1:
                    return -1
                total = np.sum(np.stack(self.bufs), axis=0, dtype=np.uint64)
                self.bar.wait(timeout=60)
                a[:] = total
                return 0
            except Exception:
                self.bar.abort()
                return -1
        return fn


def model(maps):
    names = sorted(set().union(*[set(m) for m in maps]))
    out = []
    for r in range(len(maps)):
        out.append({n: (sum(maps[q].get(n, 0) for q in range(r)), sum(m.get(n, 0) for m in maps)) for n in names})
    return out


def run_threads(maps):
    world = len(maps)
    grp = ThreadSum(world)
    cbs = [grp.for_rank(r) for r in range(world)]
    got, errs = [None] * world, [None] * world

    def one(r):
        try:
            got[r] = modkit_b200.agree_file_slices(maps[r], r, world, cbs[r] if world > 1 else None)
        except Exception as e:       # (reported below)
            errs[r] = e
    th = [threading.Thread(target=one, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert errs == [None] * world, errs
    return got, grp.calls


def random_maps(rng, world):
    pool = ["HP_%d.bed" % k for k in range(rng.randint(1, 12))] + ["ungrouped.bed", "f_0.33333334.bed", "A_missing.bed", "x" * 251 + ".bed", "p_été.bed"]
    maps = []
    for r in range(world):
        m = {}
        if rng.random() < 0.2:
            maps.append(m)            # a rank with no files at all
            continue
        for n in rng.sample(pool, rng.randint(0, len(pool))):
            m[n] = 0 if rng.random() < 0.15 else rng.choice([1, 7, 8, 9, rng.randint(1, 1 << 20), (1 << 33) + rng.randint(0, 99)])
        maps.append(m)
    return maps


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8])
def test_agreement_matches_model(world, native_lib):
    rng = random.Random(1000 + world)
    for trial in range(12):
        maps = random_maps(rng, world)
        if trial == 0:
            maps = [{} for _ in range(world)]                                 # nothing anywhere
        if trial == 1 and world > 1:
            maps = [{} for _ in range(world)]
            maps[world - 1] = {"only_last.bed": 5, "zero.bed": 0}            # names on one rank only, one of zero bytes
        got, calls = run_threads(maps)
        assert got == model(maps), (trial, maps)
        if world > 1:
            assert all(c == calls[0] for c in calls), calls          # every exchange has one length on all ranks
            assert calls[0][0] == world and len(calls[0]) == (3 if any(maps) else 1) and 0 not in calls[0]


def _gloo_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    maps = random_maps(random.Random(77), world)
    got = modkit_b200.agree_file_slices(maps[rank], rank, world, modkit_b200.torch_allreduce(None))
    dist.barrier()
    dist.destroy_process_group()
    with open(os.path.join(out, "r%d.txt" % rank), "w") as f:
        f.write(repr(sorted(got.items())) + "\n" + repr(sorted(model(maps)[rank].items())))


def test_agreement_over_gloo(native_lib, tmp_path):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_gloo_worker, args=(3, port, str(tmp_path)), nprocs=3, join=True)
    for r in range(3):
        got, want = open(tmp_path / ("r%d.txt" % r)).read().split("\n")
        assert got == want
