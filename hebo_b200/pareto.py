"""Device non-dominated filter (1 to 8 objectives, minimised) through the C ABI.

Replaces the rank-0 extraction NSGA-II performs on the final population
(HEBO/hebo/acq_optimizers/evolution_optimizer.py:141-149) for candidate batches of any size.
"""
from __future__ import annotations

from typing import Tuple

import torch

from . import _lib

_ws_cache = {}


def _workspace(dev: torch.device, need: int, tag: str = "front") -> torch.Tensor:
    key = (dev.index, tag)
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        _ws_cache[key] = ws
    return ws


def pareto_front_device(F: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """F [m,k] float32 CUDA tensor, 1 <= k <= 8 -> (idx int32 [m] whose first `count` entries are the ascending indices
    of the non-dominated rows, count int32 [1]), both on the device; NO host synchronisation.  k = 3 runs
    hb_pareto_front3, any other k hb_pareto_front_k."""
    lib = _lib.lib()
    assert F.is_cuda and F.dim() == 2 and 1 <= F.shape[1] <= _lib.HB_MAX_OBJ
    F = F.to(torch.float32).contiguous()
    m = F.shape[0]
    dev = F.device
    ws = _workspace(dev, int(lib.hb_pareto_workspace_bytes(m)))
    idx = torch.empty(m, dtype=torch.int32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    k = F.shape[1]
    with torch.cuda.device(dev):
        if k == 3:
            st = lib.hb_pareto_front3(_lib.ptr(F), m, _lib.ptr(idx), _lib.ptr(cnt), _lib.ptr(ws), ws.numel(),
                                      _lib.stream_ptr())
        else:
            st = lib.hb_pareto_front_k(_lib.ptr(F), m, k, _lib.ptr(idx), _lib.ptr(cnt), _lib.ptr(ws), ws.numel(),
                                       _lib.stream_ptr())
    _lib.check(st, "hb_pareto_front")
    return idx, cnt


def pareto_front(F: torch.Tensor) -> torch.Tensor:
    """F [m,k] float32 CUDA tensor -> ascending int64 indices (on the device) of the non-dominated rows
    (one host read of the count)."""
    idx, cnt = pareto_front_device(F)
    return idx[:int(cnt.item())].to(torch.int64)


def feasible_front(F: torch.Tensor, G: torch.Tensor) -> torch.Tensor:
    """Rank-0 set under one constraint column: F [m,k], G [m] CUDA tensors -> ascending int64 indices (on the device).
    A row is feasible iff G <= 0 (a non-finite G counts as +inf, as in hb_nsga2_survive_cv).  The result is the
    non-dominated set of the feasible rows; with no feasible row it is the single least infeasible row (smallest G, lowest
    index), which is what pymoo's filter_optimum(least_infeasible=True) is recalled to return -- not checked against
    pymoo.  Infeasible rows are masked to NaN, which the device filter already excludes."""
    G = G.reshape(-1).to(torch.float32)
    G = torch.where(torch.isfinite(G), G, torch.full_like(G, float("inf")))
    feas = G <= 0
    idx = pareto_front(torch.where(feas[:, None], F.to(torch.float32), torch.full_like(F, float("nan"), dtype=torch.float32)))
    if idx.numel() == 0 and G.numel() and not bool(feas.any()):
        idx = torch.argmin(G).reshape(1)          # first of the minima: the lowest index on ties
    return idx


FRONT_W = 8     # floats per row of a front buffer (include/hebo_b200.h "multi-GPU front exchange")


def front_pack(F: torch.Tensor, mu, var, idx: torch.Tensor, cnt: torch.Tensor, row_offset: int, capacity: int) -> torch.Tensor:
    """Fixed-capacity front buffer [(capacity + 1), 8] of the rows idx[:cnt] (hb_front_pack; no host sync)."""
    lib = _lib.lib()
    dev = F.device
    out = torch.empty(capacity + 1, FRONT_W, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        st = lib.hb_front_pack(_lib.ptr(F), _lib.ptr(mu), _lib.ptr(var), _lib.ptr(idx), _lib.ptr(cnt), int(row_offset),
                               int(capacity), _lib.ptr(out), _lib.stream_ptr())
    _lib.check(st, "hb_front_pack")
    return out


def front_merge(all_buf: torch.Tensor, world: int, capacity: int) -> torch.Tensor:
    """All-gathered buffers [world, capacity + 1, 8] -> merged front buffer [(world * capacity + 1), 8] (hb_front_merge)."""
    lib = _lib.lib()
    dev = all_buf.device
    ws = _workspace(dev, int(lib.hb_front_merge_workspace_bytes(world, capacity)), "merge")
    out = torch.empty(world * capacity + 1, FRONT_W, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        st = lib.hb_front_merge(_lib.ptr(all_buf), world, capacity, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
    _lib.check(st, "hb_front_merge")
    return out


def front_wait(buf: torch.Tensor) -> torch.Tensor:
    """Make the current stream wait for a front buffer that an overlapped exchange is still producing
    (``dist.gather_merge_fronts(overlap=True)``); a no-op for any other tensor.  Returns buf."""
    ready = getattr(buf, "_hb_ready", None)
    if ready is not None and buf.is_cuda:
        cur = torch.cuda.current_stream(buf.device)
        cur.wait_event(ready)
        buf.record_stream(cur)              # allocated on the exchange stream's pool
    return buf


def front_read(buf: torch.Tensor):
    """Host view of a front buffer: (global ids int64 [K], F [K,3], (mu, sigma) [K,2]).  This is the ONE device->host
    read of a scoring step; raises if any rank's front overflowed the gather capacity (never silently truncated)."""
    host = front_wait(buf).cpu()
    k, over = int(host[0, 0]), bool(host[0, 1] != 0)
    if over or k > host.shape[0] - 1:
        raise RuntimeError(f"local Pareto front larger than the gather capacity ({host.shape[0] - 1} rows per buffer)")
    body = host[1:k + 1]
    gid = body[:, 5].to(torch.int64) + (body[:, 6].to(torch.int64) << 24)
    return gid, body[:, :3].contiguous(), body[:, 3:5].contiguous()
