"""The two-stream chunk pipeline of hb_posterior_mace_ex.  A tensor-path call of two or more chunks runs the K* of every
chunk on the caller's stream and the contraction, guard and MACE stages on the library's highest-priority stream, with
the K* of chunk i + 1 written to the second K* / mean-partial buffer while chunk i is still contracted.  Nothing in the
arithmetic depends on that schedule, so every check here is bit for bit:
  - a call of several chunks equals one call per chunk: odd and even chunk counts, a last chunk of one row, and chunks
    where the precision guard flags rows next to chunks where it flags none;
  - two calls back to back on one workspace with no synchronisation between them equal two synchronised calls;
  - a call on a non-default torch stream is ordered before the work enqueued on that stream after it;
  - the contraction runs on a stream of its own when a call has two or more chunks, and on the caller's stream when it
    has one (kernel streams from a torch.profiler trace)."""
import ctypes as C
import json
import os
import re
import tempfile

import pytest
import torch

from hebo_b200 import _lib
from tests.test_gpu_posterior_mace import abi, guard_stats, shape_model
from tests.util import DEV

pytestmark = pytest.mark.gpu

SENTINEL = -777.25


def _off(t, row0, w=1):
    return None if t is None else C.c_void_p(t.data_ptr() + row0 * w * 4)


def enqueue(gp, Xs, m_chunk, ws, outs, seed=3):
    """One hb_posterior_mace_ex call over all rows of Xs on the current torch stream, without a synchronisation."""
    F, mu, var = outs
    lib = _lib.lib()
    st = lib.hb_posterior_mace_ex(_off(Xs, 0), None, Xs.shape[0], 0, gp.n, gp.d, C.byref(gp._spec), None, None,
                                  _off(gp._x_mul, 0), _off(gp._x_add, 0), _off(gp.Zt_dev, 0), _off(gp.alpha_dev, 0),
                                  _off(gp.Linv_dev, 0), _off(gp.Linv_hi_dev, 0), _off(gp.Linv_lo_dev, 0),
                                  _off(gp.hyp_dev, 0), gp.kern_id, gp._y_mean, float(gp._y_std), int(bool(gp.pred_likeli)),
                                  0.3, 2.0, 1e-4, None, None, seed, _off(F, 0), _off(mu, 0), _off(var, 0),
                                  C.c_void_p(ws.data_ptr()), ws.numel() * 4, m_chunk, _lib.stream_ptr())
    assert st == _lib.HB_OK, st


def outputs(m):
    return (torch.full((m, 3), SENTINEL, device=DEV), torch.full((m,), SENTINEL, device=DEV),
            torch.full((m,), SENTINEL, device=DEV))


def workspace(gp, m_chunk):
    return torch.full((int(_lib.lib().hb_posterior_workspace_bytes(gp.n, gp.d, m_chunk)) // 4,), float("nan"), device=DEV)


def per_chunk(gp, Xs, m_chunk, seed=3):
    """The reference: one synchronised single-chunk call per chunk, rng_offset = the chunk's first row."""
    m = Xs.shape[0]
    F, mu, var = outputs(m)
    ws = workspace(gp, m_chunk)
    for c0 in range(0, m, m_chunk):
        abi(gp, Xs, None, min(m_chunk, m - c0), c0, "tensor", F.view(-1), mu, var, m_chunk, seed=seed, ws=ws)
    return F, mu, var


def mixed_rows(gp, X, m, m_chunk, seed):
    """Chunk k holds rows far from the data (k % 3 == 0: the guard flags none), training rows among random rows
    (k % 3 == 1: the guard flags those) or random rows (k % 3 == 2)."""
    g = torch.Generator().manual_seed(seed)
    d = gp.d
    parts = []
    for k, c0 in enumerate(range(0, m, m_chunk)):
        mc = min(m_chunk, m - c0)
        if k % 3 == 0:
            rows = 4.0 + 2.0 * torch.rand(mc, d, generator=g)
        else:
            rows = torch.rand(mc, d, generator=g) * 2 - 1
            if k % 3 == 1:
                pick = torch.randperm(mc, generator=g)[:max(1, mc // 4)]
                rows[pick] = X[torch.randint(0, X.shape[0], (pick.numel(),), generator=g)].float()
        parts.append(rows)
    return torch.cat(parts).float().to(DEV).contiguous()


@pytest.mark.parametrize("m_chunk,m", [(512, 2 * 512 + 1), (512, 5 * 512), (384, 4 * 384 + 1), (128, 7 * 128 + 100)])
def test_chunks_equal_one_call_per_chunk(m_chunk, m):
    """3, 5, 5 and 8 chunks; the first and third cases end in a chunk of one row."""
    gp, X, _, _ = shape_model(1100)
    Xs = mixed_rows(gp, X, m, m_chunk, seed=m)
    flagged = []
    for c0 in range(0, m, m_chunk):
        guard_stats(reset=True)
        abi(gp, Xs, None, min(m_chunk, m - c0), c0, "tensor", None, outputs(m)[1], outputs(m)[2], m_chunk)
        flagged.append(guard_stats(reset=True)[1])
    print(json.dumps(dict(case="pipeline-chunks", m=m, m_chunk=m_chunk, flagged_per_chunk=flagged)))
    assert all(f == 0 for f in flagged[0::3]) and all(f > 0 for f in flagged[1::3]), flagged
    ref = per_chunk(gp, Xs, m_chunk)
    got = outputs(m)
    enqueue(gp, Xs, m_chunk, workspace(gp, m_chunk), got)
    torch.cuda.synchronize()
    for a, b in zip(ref, got):
        assert torch.equal(a, b), (m_chunk, m)


def test_back_to_back_calls_on_one_workspace():
    """Two pipelined calls on different rows share one workspace, with nothing between them: the second call's K*
    buffers are the ones the first call's last chunks read."""
    gp, X, _, _ = shape_model(1100)
    m_chunk = 512
    A = mixed_rows(gp, X, 5 * 512 + 7, m_chunk, seed=11)
    B = mixed_rows(gp, X, 4 * 512 + 300, m_chunk, seed=12)
    ws = workspace(gp, m_chunk)
    ref = []
    for Xs in (A, B):
        r = outputs(Xs.shape[0])
        enqueue(gp, Xs, m_chunk, ws, r)
        torch.cuda.synchronize()
        ref.append(r)
    got = [outputs(A.shape[0]), outputs(B.shape[0])]
    enqueue(gp, A, m_chunk, ws, got[0])
    enqueue(gp, B, m_chunk, ws, got[1])
    torch.cuda.synchronize()
    for r, g in zip(ref, got):
        for a, b in zip(r, g):
            assert torch.equal(a, b)
    for a, b in zip(ref[0], per_chunk(gp, A, m_chunk)):
        assert torch.equal(a, b)


def test_call_on_a_side_stream_orders_later_work():
    """On a non-default torch stream: a long matmul and the fill of the outputs, the call, then copies of the outputs,
    all enqueued without a synchronisation; the copies hold the call's results."""
    gp, X, _, _ = shape_model(1100)
    m_chunk, m = 512, 6 * 512 + 5
    Xs = mixed_rows(gp, X, m, m_chunk, seed=21)
    ref = per_chunk(gp, Xs, m_chunk)
    ws = workspace(gp, m_chunk)
    outs = outputs(m)
    side = torch.cuda.Stream(DEV)
    big = torch.randn(4096, 4096, device=DEV)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for _ in range(8):
            big = big @ big / 64.0
        for t in outs:
            t.fill_(SENTINEL)
        enqueue(gp, Xs, m_chunk, ws, outs)
        copies = [t.clone() for t in outs]
    side.synchronize()
    for a, b in zip(ref, copies):
        assert torch.equal(a, b)


def _kernel_streams(fn):
    """{kernel family: [stream ids]} of the CUDA kernels fn() launches, from a torch.profiler trace."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            events = json.load(fh)["traceEvents"]
    fam = {"kstar_split": re.compile(r"kstar_kernel<\d+, 2, "), "vnorm": re.compile(r"vnorm_h16_kernel"),
           "mace": re.compile(r"\bmace_kernel")}
    out = {k: [] for k in fam}
    for e in events:
        if e.get("cat") != "kernel":
            continue
        for k, rx in fam.items():
            if rx.search(e.get("name", "")):
                out[k].append(e["args"]["stream"])
    return out


def test_pipeline_is_taken_for_two_or_more_chunks_only():
    gp, X, _, _ = shape_model(1100)
    m_chunk = 512
    for m, chunks in ((m_chunk, 1), (3 * m_chunk + 1, 4)):
        Xs = mixed_rows(gp, X, m, m_chunk, seed=31)
        ws = workspace(gp, m_chunk)
        enqueue(gp, Xs, m_chunk, ws, outputs(m))     # (first use of the shape: schedule tables, stream creation)
        s = _kernel_streams(lambda: enqueue(gp, Xs, m_chunk, ws, outputs(m)))
        print(json.dumps(dict(case="pipeline-streams", m=m, chunks=chunks, streams={k: sorted(set(v)) for k, v in s.items()})))
        assert all(len(v) == chunks for v in s.values()), s
        caller, stages = set(s["kstar_split"]), set(s["vnorm"]) | set(s["mace"])
        assert len(caller) == 1 and len(stages) == 1, s
        if chunks == 1:
            assert stages == caller, s
        else:
            assert stages.isdisjoint(caller), s
