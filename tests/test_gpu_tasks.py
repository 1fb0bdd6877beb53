"""BASELINE.json configs 2-3 as parity cases (reduced sizes) plus the worker-level decode on the GPU engine. `-m gpu`.

* multi-task batch (VQA + NLVR2 + RefCOCO in thirds), sharded on pair-aligned boundaries: per-shard outputs equal the
  un-sharded ones bit for bit, and match the oracle;
* caption-image retrieval score matrix through vilbert_b200.parallel (single process = world 1) vs the oracle;
* prediction() top-k dicts from engine logits == the same decode applied to oracle logits.
"""
import pytest
import torch

import support

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine(full_oracle):
    yield from support.one_engine(full_oracle)


def test_multitask_batch_sharded(full_oracle, engine, parity_log):
    """configs[2] at B=24: task tokens 1 (VQA) / 12 (NLVR2, adjacent pairs) / 11 (RefCOCO) in thirds; 3 pair-aligned shards."""
    from oracle import vilbert_ref as R
    from vilbert_b200 import parallel as P
    B = 24
    inp = list(R.make_inputs(B, 30, 36, seed=555, pad_regions=2))
    task = torch.cat([torch.full((8, 1), 1), torch.full((8, 1), 12), torch.full((8, 1), 11)]).long()
    inp[7] = task
    ref = full_oracle(*inp, compute_pretraining_heads=False)
    dev = [t.cuda() for t in inp]
    whole = engine(*dev)
    torch.cuda.synchronize()
    for i, name in ((0, "vil_prediction"), (3, "vil_binary_prediction"), (6, "vision_logit")):
        r, o = ref[i], whole[i].cpu()
        small = r.abs() < 1000
        err = float((o - r).abs()[small].max())
        parity_log(test="multitask_B24", output=name, max_abs_err=err)
        assert err < 1e-2, (name, err)
    world = 3
    outs = []
    for rank in range(world):
        lo, hi = P.shard_range(B, rank, world, pair_aligned=True)
        assert lo % 2 == 0 and hi % 2 == 0
        outs.append(engine(*[t[lo:hi] for t in dev]))
    torch.cuda.synchronize()
    assert torch.equal(torch.cat([o[0] for o in outs]), whole[0])
    assert torch.equal(torch.cat([o[3] for o in outs]), whole[3])          # NLVR2 pairs never straddle a shard
    assert torch.equal(torch.cat([o[6] for o in outs]), whole[6])


def test_retrieval_score_matrix(full_oracle, engine, parity_log):
    """configs[3] at 6 captions x 5 images: score[c, i] = vil_logit of pair (c, i), task token 7 (worker.py:278-284, 359)."""
    from oracle import vilbert_ref as R
    from vilbert_b200 import parallel as P
    n_cap, n_img = 6, 5
    cap = R.make_inputs(n_cap, 30, 36, seed=901)
    img = R.make_inputs(n_img, 30, 36, seed=902)
    q, seg, im = cap[0], cap[3], cap[4]
    f, s, vm = img[1], img[2], img[5]
    ref = torch.empty(n_cap, n_img)
    for c in range(n_cap):
        out = full_oracle(q[c:c + 1].repeat(n_img, 1), f, s, seg[c:c + 1].repeat(n_img, 1), im[c:c + 1].repeat(n_img, 1), vm,
                          None, torch.full((n_img, 1), 7), compute_pretraining_heads=False)
        ref[c] = out[2].view(-1)
    score = P.make_pair_scorer(engine, (q.cuda(), seg.cuda(), im.cuda()), (f.cuda(), s.cuda(), vm.cuda()))
    full = P.retrieval_scores(score, n_cap, n_img, image_chunk=3).cpu()
    err = float((full - ref).abs().max())
    parity_log(test="retrieval_6x5", max_abs_err=err, ref_std=float(ref.std()))
    assert full.shape == (n_cap, n_img) and err < 1e-2
    # ranking of the images per caption is what the worker returns (worker.py:359-366)
    assert torch.equal(full.argmax(1), ref.argmax(1))


@pytest.mark.parametrize("task_id,n_img", [("1", 1), ("15", 1), ("12", 2), ("13", 1), ("7", 3), ("11", 1)])
def test_prediction_on_engine_matches_oracle_decode(full_oracle, engine, task_id, n_img):
    """worker.prediction() driven by the engine returns the dict the same decode gives on the oracle's logits."""
    from oracle import vilbert_ref as R
    from vilbert_b200 import worker_api as W
    W.model = engine
    inp = R.make_inputs(n_img, 37, 20, seed=77 + n_img)
    text, segs, mask = inp[0][:1], inp[3][:1], inp[4][:1]
    task = torch.tensor([[int(task_id)]])
    infos = [{"image_width": 640, "image_height": 480}] * n_img
    ans = W.prediction(text.cuda(), inp[1].cuda(), inp[2].cuda(), segs.cuda(), mask.cuda(), inp[5].cuda(), inp[6].cuda(),
                       task.cuda(), task_id, infos)

    class OracleAsModel:
        _device = 0

        def __call__(self, *a, **kw):
            kw.pop("select", None)
            a = [t.cpu() if torch.is_tensor(t) else t for t in a]
            return full_oracle(*a, compute_pretraining_heads=False)
    W.model = OracleAsModel()
    ref = W.prediction(text, inp[1], inp[2], segs, mask, inp[5], inp[6], task, task_id, infos)
    W.model = engine
    if isinstance(ans, list):
        assert [(a["x1"], a["y1"], a["x2"], a["y2"]) for a in ans] == [(a["x1"], a["y1"], a["x2"], a["y2"]) for a in ref]
        assert [a["confidence"] for a in ans] == pytest.approx([a["confidence"] for a in ref], abs=0.5)
    else:
        assert ans["top3_answer"] == ref["top3_answer"]
        assert ans["top3_confidence"] == pytest.approx(ref["top3_confidence"], abs=5e-3)


def test_multitask_b512_full_size_properties(full_oracle, engine, parity_log):
    """BASELINE.json configs[2] at its full size (B = 512, 64 per GPU on 8 GPUs, task tokens VQA / NLVR2 / RefCOCO in thirds,
    NLVR2 samples as adjacent pairs).  Size-independent properties: the eight pair-aligned rank slices reproduce the whole-batch
    outputs bit for bit, and sampled rows match the oracle (which only sees those rows -- pairs are independent)."""
    from oracle import vilbert_ref as R
    from vilbert_b200 import parallel as P
    B, world = 512, 8
    inp = list(R.make_inputs(B, 30, 36, seed=4242, pad_regions=1))
    n3 = (B // 3) // 2 * 2                                    # thirds on pair boundaries: 170 / 170 / 172
    task = torch.cat([torch.full((n3, 1), 1), torch.full((n3, 1), 12), torch.full((B - 2 * n3, 1), 11)]).long()
    inp[7] = task
    dev = [t.cuda() for t in inp]
    whole = engine(*dev)
    torch.cuda.synchronize()
    whole = [w.clone() if torch.is_tensor(w) else w for w in whole]
    for rank in range(world):
        lo, hi = P.shard_range(B, rank, world, pair_aligned=True)
        assert (lo, hi) == (64 * rank, 64 * rank + 64)
        out = engine(*[t[lo:hi] for t in dev])
        torch.cuda.synchronize()
        assert torch.equal(out[0], whole[0][lo:hi])
        assert torch.equal(out[3], whole[3][lo // 2:hi // 2])
        assert torch.equal(out[6], whole[6][lo:hi])
    rows = [0, 1, n3, n3 + 1, 2 * n3, 2 * n3 + 1, B - 2, B - 1]          # pairs (2i, 2i+1) stay together
    ref = full_oracle(*[t[rows] for t in inp], compute_pretraining_heads=False)
    errs = {}
    for i, name in ((0, "vil_prediction"), (6, "vision_logit")):
        r, o = ref[i], whole[i][rows].cpu()
        small = r.abs() < 1000
        errs[name] = float((o - r).abs()[small].max())
    pair_rows = [r // 2 for r in rows[::2]]
    errs["vil_binary_prediction"] = float((whole[3][pair_rows].cpu() - ref[3]).abs().max())
    for name, err in errs.items():
        parity_log(test="multitask_B512", output=name, max_abs_err=err)
        assert err < 1e-2, (name, err)


def test_retrieval_1000x1000_rank_block(full_oracle, engine, parity_log):
    """BASELINE.json configs[3] at its full size as ONE rank of eight sees it: 125 of 1000 captions against all 1000 images
    (125 k pair forwards).  Properties: the block does not depend on how the images are chunked into forwards (bit-exact),
    and sampled entries match the oracle's vil_logit of that (caption, image) pair."""
    from oracle import vilbert_ref as R
    from vilbert_b200 import parallel as P
    n_cap, n_img, world, rank = 1000, 1000, 8, 3
    lo, hi = P.shard_range(n_cap, rank, world)
    assert hi - lo == 125
    g = torch.Generator().manual_seed(7007)
    cap = R.make_inputs(hi - lo, 30, 36, seed=7100 + rank)            # this rank's captions
    base = R.make_inputs(50, 30, 36, seed=7200)                       # 1000 images = 50 distinct feature sets x 20 variants
    f = base[1].repeat(20, 1, 1) * (0.75 + 0.5 * torch.rand(n_img, 1, 1, generator=g))
    s, vm = base[2].repeat(20, 1, 1), base[5].repeat(20, 1)
    q, seg, im = cap[0], cap[3], cap[4]
    score = P.make_pair_scorer(engine, (q.cuda(), seg.cuda(), im.cuda()), (f.cuda(), s.cuda(), vm.cuda()))
    block = torch.stack([torch.cat([score(c, torch.arange(a, min(n_img, a + 250))).reshape(-1).float()
                                    for a in range(0, n_img, 250)]) for c in range(hi - lo)])
    torch.cuda.synchronize()
    assert block.shape == (125, n_img) and torch.isfinite(block).all()
    for c in (0, 57, 124):                                            # other chunkings of the image axis: same bits
        again = torch.cat([score(c, torch.arange(a, min(n_img, a + 64))).reshape(-1).float() for a in range(0, n_img, 64)])
        assert torch.equal(again, block[c])
    picks = [(0, 0), (3, 999), (57, 500), (124, 123), (99, 731), (64, 64)]
    worst = 0.0
    for c, i in picks:
        out = full_oracle(q[c:c + 1], f[i:i + 1], s[i:i + 1], seg[c:c + 1], im[c:c + 1], vm[i:i + 1], None, torch.full((1, 1), 7),
                          compute_pretraining_heads=False)
        worst = max(worst, abs(float(out[2].view(-1)[0]) - float(block[c, i])))
    parity_log(test="retrieval_1000x1000_rank_block", max_abs_err=worst, ref_std=float(block.std()))
    assert worst < 1e-2
    # round 2: the same block with reuse (caption prefix once per caption, image prefix once per image, connection layers per
    # pair): bit-identical, and faster (19 % fewer FLOPs plus no per-call text repeat / feature gather on the host side)
    import time
    caps, imgs = (q.cuda(), seg.cuda(), im.cuda()), (f.cuda(), s.cuda(), vm.cuda())
    P.retrieval_scores_cached(engine, tuple(t[:2] for t in caps), imgs, pair_batch=250)      # plans built outside the timing
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tm = {}
    cached = P.retrieval_scores_cached(engine, caps, imgs, pair_batch=250, timings=tm)
    torch.cuda.synchronize()
    t_cached = time.perf_counter() - t0
    assert torch.equal(cached.cpu(), block.cpu())
    t0 = time.perf_counter()
    for c in range(hi - lo):
        for a in range(0, n_img, 250):
            score(c, torch.arange(a, min(n_img, a + 250)))
    torch.cuda.synchronize()
    t_plain = time.perf_counter() - t0
    parity_log(test="retrieval_1000x1000_rank_block_cached", seconds_cached=t_cached, seconds_plain=t_plain,
               speedup=t_plain / t_cached, **{k: float(v) for k, v in tm.items()})
    assert t_cached < 0.87 * t_plain, (t_cached, t_plain)


def test_prediction_batch_on_engine_is_exact(full_oracle, engine):
    """Micro-batched requests (worker_api.prediction_batch: one forward for all of them, NLVR2 on even rows) decode to exactly
    what one-request-at-a-time prediction() returns -- the engine's rows do not depend on their batch neighbours."""
    from oracle import vilbert_ref as R
    from vilbert_b200 import worker_api as W
    W.model = engine
    W.label_maps.update(vqa=None, gqa=None)
    reqs = []
    for k, (task_id, n_img) in enumerate([("1", 1), ("12", 2), ("7", 3), ("11", 1), ("13", 1), ("15", 1), ("12", 2), ("4", 1)]):
        inp = R.make_inputs(n_img, 37, 20, seed=300 + k)
        reqs.append((inp[0][:1].cuda(), inp[1].cuda(), inp[2].cuda(), inp[3][:1].cuda(), inp[4][:1].cuda(), inp[5].cuda(),
                     inp[6].cuda(), torch.tensor([[int(task_id)]]).cuda(), task_id,
                     [{"image_width": 640, "image_height": 480}] * n_img))
    single = [W.prediction(*r) for r in reqs]
    got = W.prediction_batch(reqs)
    for a, b in zip(got, single):
        if isinstance(a, list):
            assert a == b
        else:
            assert a["top3_answer"] == b["top3_answer"] and a["top3_confidence"] == b["top3_confidence"]
