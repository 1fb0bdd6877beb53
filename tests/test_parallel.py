"""Host-side multi-GPU logic on CPU: sharding arithmetic, and a world_size-2 gloo run of the retrieval
all-gather and of batch-sharded execution (the N>1 path of bench.py / vilbert_b200.parallel)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from vilbert_b200 import parallel as P
import support


def test_shard_range_covers_and_balances():
    for n in (0, 1, 7, 64, 125, 512, 1000):
        for world in (1, 2, 3, 8):
            spans = [P.shard_range(n, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            sizes = [hi - lo for lo, hi in spans]
            assert max(sizes) - min(sizes) <= 1


def test_shard_range_pair_aligned():
    for n in (2, 10, 64, 170, 512):
        for world in (1, 2, 3, 8):
            spans = [P.shard_range(n, r, world, pair_aligned=True) for r in range(world)]
            assert spans[-1][1] == n and all(lo % 2 == 0 and hi % 2 == 0 for lo, hi in spans)
    with pytest.raises(ValueError):
        P.shard_range(7, 0, 2, pair_aligned=True)


def _worker(rank, world, port, n_cap, n_img, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(0)
        table = torch.randn(n_cap, n_img, generator=g)          # "model": score of (caption c, image i)
        calls = []

        def score(c, idx):
            calls.append((c, idx.numel()))
            return table[c, idx].unsqueeze(1)

        full = P.retrieval_scores(score, n_cap, n_img, image_chunk=4)
        lo, hi = P.shard_range(n_cap, rank, world)
        ok = torch.equal(full, table) and {c for c, _ in calls} == set(range(lo, hi))
        # batch-sharded "forward": each rank handles its slice; gathered result == single-process result
        x = torch.arange(22, dtype=torch.float32).view(11, 2)
        mine = P.shard_batch([x], rank, world)[0] * 2.0
        ok = ok and torch.equal(P.all_gather_rows(mine, 11), x * 2.0)
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("n_cap,n_img", [(5, 6), (8, 10)])
def test_retrieval_allgather_gloo_world2(n_cap, n_img):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = support.free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, n_cap, n_img, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert res == [(0, True), (1, True)]


def test_single_process_paths():
    t = torch.randn(3, 4)
    assert P.all_gather_rows(t, 3) is t
    full = P.retrieval_scores(lambda c, idx: torch.full((idx.numel(), 1), float(c)), 3, 5, image_chunk=2)
    assert full.shape == (3, 5) and torch.equal(full[:, 0], torch.tensor([0.0, 1.0, 2.0]))
