// Tile geometry and host-built tile schedule of the posterior variance contraction (vnorm_h16.cu).  Plain C++ so that
// the schedule's invariants can be checked without a GPU (tests/test_vnorm_schedule.py).
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

namespace hb {
namespace h16 {

constexpr int BM = 128;            // candidates per tile (two consumer warpgroups of 64)
constexpr int BN = 128;            // Linv rows per tile (wgmma N)
constexpr int BK = 64;             // fp16 elements per k-block = one 128-byte swizzle row
// CTAs per cluster: they share every Linv box by TMA multicast, so a k-block moves 32 KiB of K* + 32 / CLUSTER KiB of
// Linv per CTA from L2.  4 rather than 2: only 30 clusters of 4 fit on a 132-SM H100 SXM (120 CTAs, against 66 pairs),
// yet the contraction measured 3 % faster and the scoring step 5-6 % faster than with pairs (H100 80GB HBM3, 400 W power
// limit: the idle SMs and the lighter L2 traffic leave the power-capped clock higher).
constexpr int CLUSTER = 4;

// Tile schedule: one list per cluster (codes p << 16 | J, terminated by -1).  A unit (p, J) is the column tile J of the
// CLUSTER bands rt = CLUSTER p + rank, one per CTA of the cluster; the CTAs of a cluster walk the same J sequence, so they
// need the same Linv boxes in the same order, and each loads 1 / CLUSTER of them for all.  An n_rt that is not a multiple
// of CLUSTER is padded with bands whose rows lie beyond the chunk (the caller's workspace holds them; nothing reads their
// results).  Units are handed out in BAND-MAJOR order -- all column tiles J of one band group, heaviest (longest k range)
// first, before the next group -- to whichever cluster is least loaded at that point (a simulation of a dynamic scheduler
// with the k-block count + an epilogue allowance as the cost; the last groups are dealt heaviest-first ACROSS groups so
// that the lists end with cheap units).  Two effects: the clusters finish within a few per cent of each other, and the
// CTAs working on one band at the same time read its K* rows once from HBM and then from L2, instead of streaming the
// whole K* chunk once per column tile.
// Returns the flat table [clusters][*len] the kernel reads.
inline std::vector<int32_t> build_schedule(int np, int n_rt, int clusters, int *len) {
  const int n_j = (np + BN - 1) / BN;
  const int n_p = (n_rt + CLUSTER - 1) / CLUSTER;
  constexpr int EPI_COST = 1;   // epilogue in k-block units (a register drain and one shuffle reduction per tile)
  std::vector<std::vector<int32_t>> lists(clusters);
  std::vector<long long> load(clusters, 0);
  // band-major body, then the units of the last TAIL_BANDS bands heaviest-first across bands (an LPT tail: the list ends
  // with the cheapest units, which levels the clusters instead of leaving one heavy unit of overhang)
  constexpr int TAIL_BANDS = 16;
  const int body = std::max(0, n_p - TAIL_BANDS / CLUSTER);
  auto give = [&](int p, int J) {
    int best = 0;
    for (int c = 1; c < clusters; ++c)
      if (load[c] < load[best]) best = c;
    const int kend = std::min((J + 1) * BN, np);
    load[best] += kend / BK + EPI_COST;
    lists[best].push_back((p << 16) | J);
  };
  for (int p = 0; p < body; ++p)
    for (int J = n_j - 1; J >= 0; --J) give(p, J);
  for (int J = n_j - 1; J >= 0; --J)
    for (int p = body; p < n_p; ++p) give(p, J);
  size_t l = 0;
  for (auto &x : lists) l = std::max(l, x.size());
  l += 1;
  std::vector<int32_t> flat((size_t)clusters * l, -1);
  for (int c = 0; c < clusters; ++c) std::copy(lists[c].begin(), lists[c].end(), flat.begin() + (size_t)c * l);
  *len = (int)l;
  return flat;
}

}  // namespace h16
}  // namespace hb
