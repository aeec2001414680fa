"""Host-only checks of the tile schedule of the posterior variance contraction (hebo_b200/csrc/vnorm_sched.h).

The kernel reads one list per cluster of CLUSTER CTAs; the CTA of rank r runs band rt = CLUSTER * p + r of every unit
(p, J).  A tile the schedule drops leaves stale partial sums behind, a tile it repeats is counted twice, and two CTAs of a
cluster that disagree on J wait forever for each other's multicast -- so every chunk shape must be covered exactly."""
import os
import shutil
import subprocess

import numpy as np
import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hebo_b200", "csrc")

DRIVER = r"""
#include <cstdio>
#include "vnorm_sched.h"
int main() {
  int np, n_rt, clusters;
  std::printf("%d %d %d %d\n", hb::h16::CLUSTER, hb::h16::BM, hb::h16::BN, hb::h16::BK);
  while (std::scanf("%d %d %d", &np, &n_rt, &clusters) == 3) {
    int len = 0;
    const std::vector<int32_t> t = hb::h16::build_schedule(np, n_rt, clusters, &len);
    std::printf("%d", len);
    for (int32_t c : t) std::printf(" %d", c);
    std::printf("\n");
  }
}
"""


@pytest.fixture(scope="module")
def schedule(tmp_path_factory):
    cxx = shutil.which("c++") or shutil.which("g++")
    assert cxx, "a host C++ compiler is needed to build the schedule driver"
    d = tmp_path_factory.mktemp("sched")
    src, exe = d / "driver.cpp", d / "driver"
    src.write_text(DRIVER)
    subprocess.run([cxx, "-std=c++17", "-O1", "-I", CSRC, str(src), "-o", str(exe)], check=True)

    def run(shapes):
        out = subprocess.run([str(exe)], input="".join(f"{a} {b} {c}\n" for a, b, c in shapes), capture_output=True,
                             text=True, check=True).stdout.splitlines()
        geom = tuple(int(x) for x in out[0].split())
        tables = []
        for (np_, n_rt, clusters), line in zip(shapes, out[1:]):
            v = np.array(line.split(), dtype=np.int64)
            tables.append(v[1:].reshape(clusters, int(v[0])))
        return geom, tables
    return run


def _clusters(n_rt, n_j, cluster, max_clusters):
    return min(max_clusters, -(-n_rt // cluster) * n_j)


def _shapes():
    # np: the padded training-set sizes of the tests and the bench (n = 150 ... 4096 -> multiples of 128); n_rt: the
    # 128-candidate bands of a chunk, from one row to the bench's 32 768-candidate chunk (256 bands), its 10 000-candidate
    # suggest() batch (79) and the odd / non-multiple-of-cluster counts between; grids of 66 clusters (132 SMs in pairs),
    # 30 (clusters of 4 on an H100 SXM) and smaller
    shapes = []
    for np_ in (128, 256, 384, 512, 1024, 2048, 4096):
        n_j = np_ // 128
        for n_rt in list(range(1, 20)) + [31, 32, 33, 63, 64, 65, 79, 127, 128, 129, 255, 256]:
            for max_clusters in (66, 30, 7, 1):
                shapes.append((np_, n_rt, max_clusters))
    return shapes


def test_every_tile_of_every_chunk_shape_is_scheduled_exactly_once(schedule):
    shapes = _shapes()
    (cluster, bm, bn, bk), _ = schedule([])
    assert bm == bn == 128 and bk == 64 and cluster >= 1
    calls = [(np_, n_rt, _clusters(n_rt, np_ // bn, cluster, mc)) for np_, n_rt, mc in shapes]
    _, tables = schedule(calls)
    for (np_, n_rt, clusters), t in zip(calls, tables):
        n_j = np_ // bn
        n_p = -(-n_rt // cluster)
        assert t.shape[0] == clusters and (t[:, -1] == -1).all()
        seen = np.zeros((n_p * cluster, n_j), dtype=np.int64)
        loads = []
        for lst in t:
            valid = lst[lst >= 0]
            # a list is a prefix of codes, then only the -1 terminator padding: the kernel stops at the first -1
            assert (lst[len(valid):] == -1).all(), (np_, n_rt, clusters)
            p, J = valid >> 16, valid & 0xFFFF
            assert ((p >= 0) & (p < n_p) & (J >= 0) & (J < n_j)).all()
            # what the CTAs of the cluster run: same J sequence, neighbouring bands
            per_rank = [(cluster * p + r, J) for r in range(cluster)]
            for r in range(1, cluster):
                assert np.array_equal(per_rank[r][1], per_rank[0][1])
            for rt, j in per_rank:
                np.add.at(seen, (rt, j), 1)
            loads.append(int(np.minimum((J + 1) * bn, np_).sum() // bk + J.size))
        assert (seen == 1).all(), (np_, n_rt, clusters)   # every real tile once; the padding bands of the last cluster once
        assert seen.shape[0] - n_rt < cluster
        # the greedy deal keeps the clusters level: no list exceeds the mean by more than one heaviest unit
        assert max(loads) - sum(loads) / len(loads) <= n_j * bn // bk + 1, (np_, n_rt, clusters, loads)


def test_the_bench_chunk_gives_every_cluster_work_band_major(schedule):
    """n = 4096, one 32 768-candidate chunk on 30 clusters: the K* band each cluster works on advances together
    (band-major), so the rows of a band are read from HBM about once."""
    _, (t,) = schedule([(4096, 256, 30)])
    p = [lst[lst >= 0] >> 16 for lst in t]
    assert all(len(x) > 0 for x in p)
    for x in p:
        assert (np.diff(x[: len(x) // 2]) >= 0).all()     # the body of every list walks the bands in order
