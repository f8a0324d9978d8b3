"""CPU tier: the N>1 host path on gloo, world_size 2 — SyncBN statistics exchange/merge and bench timing
reduction. (The kernels need a GPU; what is covered here is the rank plumbing around them.)"""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.torch_oracle import merge_moments


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from semseg_b200.dist_utils import gather_rank_stats, max_over_ranks, shard_batch
    try:
        rng = np.random.default_rng(0)
        full = (rng.standard_normal((8, 50, 16)) * 3 + 1.5).astype(np.float64)   # [images, pixels, C]
        mine = full[list(shard_batch(8, world, rank))].reshape(-1, 16)
        local = np.stack([mine.mean(0), ((mine - mine.mean(0)) ** 2).sum(0), np.full(16, mine.shape[0], float)])
        g = gather_rank_stats(torch.from_numpy(local))
        assert tuple(g.shape) == (world, 3, 16)
        mean, m2, n = merge_moments([(g[r, 0].numpy(), g[r, 1].numpy(), g[r, 2].numpy()) for r in range(world)])
        allx = full.reshape(-1, 16)
        ok = np.allclose(mean, allx.mean(0), atol=1e-12) and np.allclose(m2 / n, allx.var(0), atol=1e-12)
        ok = ok and bool((n == allx.shape[0]).all())
        t = max_over_ranks(1.0 + rank, "cpu")
        ok = ok and t == float(world)
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_syncbn_stats_exchange_and_timing_reduce_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(60)
    assert sorted(res) == [(0, True), (1, True)]


def test_peer_exchange_slot_sequence_and_nccl_override(monkeypatch):
    """Host logic of the NVLink peer exchange: slots advance identically on every rank and a slot is only reused with a
    strictly larger sequence number (the step counter); SEMSEG_B200_SYNCBN=nccl disables the peer path."""
    from semseg_b200 import p2p

    class Fake(p2p.PeerExchange):
        def __init__(self):
            self.calls = 0
            self.step = torch.ones((1,), dtype=torch.int32)      # the device-resident step counter (CPU stand-in)
    a, b = Fake(), Fake()
    seen = {}
    for k in range(3 * p2p.N_SLOTS + 5):
        if k % 200 == 199:          # a training forward opens a new epoch on every rank at the same point
            a.begin_step(), b.begin_step()
        slot = a.next()
        assert slot == b.next() and int(a.step) == int(b.step)
        assert 0 <= slot < p2p.N_SLOTS
        assert int(a.step) > seen.get(slot, 0)          # a slot is only reused under a larger sequence number
        seen[slot] = int(a.step)
    assert p2p.SLOT_FLOATS >= 3 * 2048          # widest BatchNorm on the path (layer4 / PSA proj: 2048 channels)
    monkeypatch.setenv("SEMSEG_B200_SYNCBN", "nccl")
    assert p2p.get_exchange(object()) is None
    assert p2p.exchange_kind() == "none"        # no process group initialised in this process


def _log_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from semseg_b200.train_utils import reduce_step_logging
    try:
        k = 7
        g = torch.Generator().manual_seed(rank)
        ml, al = torch.rand((), generator=g) + 1, torch.rand((), generator=g) + 1
        loss = ml + 0.4 * al
        n = 3 + rank
        inter, union, tgt = (torch.randint(0, 50, (k,), generator=g).float() for _ in range(3))
        # the reference's seven all-reduces (tool/train.py:280-288)
        r_ml, r_al, r_loss = ml * n, al * n, loss * n
        cnt = torch.tensor([n], dtype=torch.long)
        ri, ru, rt = inter.clone(), union.clone(), tgt.clone()
        for t in (r_ml, r_al, r_loss, cnt, ri, ru, rt):
            dist.all_reduce(t)
        m = reduce_step_logging(ml, al, loss, n, inter, union, tgt)
        ok = (torch.allclose(m.main_loss, r_ml / cnt.item(), rtol=1e-6) and torch.allclose(m.aux_loss, r_al / cnt.item(), rtol=1e-6)
              and torch.allclose(m.loss, r_loss / cnt.item(), rtol=1e-6) and int(m.n) == cnt.item()
              and torch.equal(m.intersection, ri) and torch.equal(m.union, ru) and torch.equal(m.target, rt))
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_step_logging_single_allreduce_matches_the_references_seven_world2():
    """SURVEY §8 f4: one packed all-reduce == the reference's seven (tool/train.py:278-289), world size 2 on gloo."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_log_worker, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = [q.get(timeout=120) for _ in procs]
    for p_ in procs:
        p_.join(60)
    assert sorted(res) == [(0, True), (1, True)]
