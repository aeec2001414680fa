"""CPU tests (gloo, world_size 2) of the candidate-sharding host protocol in hebo_b200/dist.py: shard bounds,
fixed-capacity front buffers, the one all-gather, merge, overflow detection at read time.  Scoring, the dominance
filter and the pack / merge steps are injected as torch restatements of the CUDA entry points (the oracle's numpy
filter stands in for the device kernel; tests/test_gpu_parity.py checks the CUDA pack / merge against the same
restatements), so no GPU is needed."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from hebo_b200 import dist as hdist
from hebo_b200.pareto import FRONT_W, front_read
from oracle import gp_oracle as O


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def front_fn_torch(F):
    """(idx padded int32 [m], count int32 [1]) like hb_pareto_front3."""
    keep = torch.from_numpy(O.pareto_front(F.numpy()))
    idx = torch.zeros(F.shape[0], dtype=torch.int32)
    idx[:keep.numel()] = keep.to(torch.int32)
    return idx, torch.tensor([keep.numel()], dtype=torch.int32)


def pack_fn_torch(F, mu, var, idx, cnt, row_offset, capacity):
    """include/hebo_b200.h hb_front_pack, restated."""
    k = int(cnt[0])
    buf = torch.zeros(capacity + 1, FRONT_W)
    buf[1:, :3] = float("inf")
    buf[0, 0], buf[0, 1] = float(k), float(k > capacity)
    kk = min(k, capacity)
    rows = idx[:kk].long()
    gid = rows + row_offset
    buf[1:kk + 1, :3] = F[rows]
    buf[1:kk + 1, 3] = mu[rows]
    buf[1:kk + 1, 4] = var[rows].sqrt()
    buf[1:kk + 1, 5] = (gid & 0xFFFFFF).float()
    buf[1:kk + 1, 6] = (gid >> 24).float()
    return buf


def merge_fn_torch(all_buf, world, capacity):
    """include/hebo_b200.h hb_front_merge, restated."""
    counts = all_buf[:, 0, 0].long()
    over = bool((counts > capacity).any()) or bool((all_buf[:, 0, 1] != 0).any())
    body = all_buf[:, 1:, :].reshape(world * capacity, FRONT_W)
    valid = (torch.arange(capacity)[None, :] < counts.clamp(max=capacity)[:, None]).reshape(-1)
    # rows beyond a rank's count are NaN, which the filter excludes: +inf rows would not dominate one another
    Fm = torch.where(valid[:, None], body[:, :3], torch.full_like(body[:, :3], float("nan")))
    keep = torch.from_numpy(O.pareto_front(Fm.numpy()))
    out = torch.zeros(world * capacity + 1, FRONT_W)
    out[1:, :3] = float("inf")
    out[0, 0], out[0, 1] = float(keep.numel()), float(over)
    out[1:keep.numel() + 1] = body[keep]
    return out


def _fake_objectives(m, seed=0):
    g = torch.Generator().manual_seed(seed)
    F = torch.randn(m, 3, generator=g)
    F[:, 2] = 0.5 * F[:, 0] + 0.5 * F[:, 2]
    mu = torch.randn(m, generator=g)
    var = torch.rand(m, generator=g) + 0.1
    return F, mu, var


def _worker(rank, world, port, m, capacity, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        F, mu, var = _fake_objectives(m)
        lo, hi = hdist.shard_bounds(m, world, rank)

        def score_fn(x):           # x carries the row ids of this shard
            ids = x.reshape(-1).long()
            return F[ids], mu[ids], var[ids]
        rows = torch.arange(lo, hi, dtype=torch.float32).reshape(-1, 1)
        buf = hdist.sharded_score_front(None, rows, lo, 0.0, 1.0, capacity=capacity, score_fn=score_fn,
                                        front_fn=front_fn_torch, pack_fn=pack_fn_torch, merge_fn=merge_fn_torch,
                                        overlap=(rank == 0))       # host tensors: the flag is ignored, no rank may diverge
        assert buf.shape == (world * capacity + 1, FRONT_W)
        try:
            gidx, Ff, extra = front_read(buf)
            np.savez(os.path.join(out_dir, f"r{rank}.npz"), idx=gidx.numpy(), F=Ff.numpy(), extra=extra.numpy(), err=0)
        except RuntimeError as e:
            np.savez(os.path.join(out_dir, f"r{rank}.npz"), err=1, msg=str(e))
    finally:
        dist.destroy_process_group()


def test_shard_bounds_cover_exactly():
    for m, w in [(10, 3), (8, 8), (1048576, 8), (5, 8)]:
        b = [hdist.shard_bounds(m, w, r) for r in range(w)]
        assert b[0][0] == 0 and b[-1][1] == m
        assert all(b[i][1] == b[i + 1][0] for i in range(w - 1))
        assert max(h - l for l, h in b) - min(h - l for l, h in b) <= 1


@pytest.mark.timeout(120)
def test_two_rank_gather_merge_equals_global_front(tmp_path):
    m = 5000
    mp.spawn(_worker, args=(2, _free_port(), m, 512, str(tmp_path)), nprocs=2, join=True)
    F, mu, var = _fake_objectives(m)
    ref = O.pareto_front(F.numpy())
    r0, r1 = np.load(tmp_path / "r0.npz"), np.load(tmp_path / "r1.npz")
    assert int(r0["err"]) == 0 and int(r1["err"]) == 0
    assert np.array_equal(r0["idx"], ref) and np.array_equal(r1["idx"], ref)      # identical on every rank
    assert np.array_equal(r0["F"], F.numpy()[ref])
    np.testing.assert_allclose(r0["extra"][:, 0], mu.numpy()[ref])
    np.testing.assert_allclose(r0["extra"][:, 1], np.sqrt(var.numpy()[ref]), rtol=1e-6)


@pytest.mark.timeout(120)
def test_front_overflow_is_reported_not_truncated(tmp_path):
    mp.spawn(_worker, args=(2, _free_port(), 5000, 2, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(tmp_path / "r0.npz"), np.load(tmp_path / "r1.npz")
    assert int(r0["err"]) == 1 and int(r1["err"]) == 1 and "capacity" in str(r0["msg"])


def test_single_process_path_is_the_local_buffer():
    F, mu, var = _fake_objectives(300)
    idx, cnt = front_fn_torch(F)
    buf = pack_fn_torch(F, mu, var, idx, cnt, 100, 64)
    out = hdist.gather_merge_fronts(buf, 64, merge_fn_torch)
    gidx, Ff, extra = front_read(out)
    ref = O.pareto_front(F.numpy())
    assert np.array_equal(gidx.numpy(), ref + 100) and torch.equal(Ff, F[ref])
    # ids above 2^24 survive the two-halves encoding
    buf2 = pack_fn_torch(F, mu, var, idx, cnt, (1 << 30) + 5, 64)
    assert np.array_equal(front_read(buf2)[0].numpy(), ref + (1 << 30) + 5)


def _rank_buffers(counts, capacity, m=400, offset_step=1000):
    """One packed buffer per rank whose local front has counts[r] rows (0: every objective of the shard is NaN)."""
    bufs = []
    for r, want in enumerate(counts):
        F, mu, var = _fake_objectives(m, seed=r + 1)
        idx, cnt = front_fn_torch(F)
        if want == 0:
            F = torch.full_like(F, float("nan"))
            idx, cnt = front_fn_torch(F)
            assert int(cnt[0]) == 0
        bufs.append(pack_fn_torch(F, mu, var, idx, cnt, r * offset_step, capacity))
    return torch.stack(bufs)


def test_merge_of_empty_fronts_is_empty():
    """Ranks whose local fronts are all empty merge to an empty front, not to world * capacity padding rows."""
    for world, capacity in ((2, 4), (8, 64)):
        out = merge_fn_torch(_rank_buffers([0] * world, capacity), world, capacity)
        assert int(out[0, 0]) == 0 and int(out[0, 1]) == 0
        gidx, Ff, extra = front_read(out)
        assert gidx.numel() == 0 and Ff.shape == (0, 3)


def test_merge_ignores_empty_ranks():
    """A merge in which some ranks are empty equals the merge of the non-empty ranks alone."""
    capacity = 256
    all_buf = _rank_buffers([1, 0, 1, 0], capacity)
    full = merge_fn_torch(all_buf, 4, capacity)
    part = merge_fn_torch(all_buf[[0, 2]], 2, capacity)
    assert int(full[0, 0]) == int(part[0, 0]) > 0
    for a, b in zip(front_read(full), front_read(part)):
        assert torch.equal(a, b)
