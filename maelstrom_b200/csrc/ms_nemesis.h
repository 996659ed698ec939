// ms_nemesis.h -- the arithmetic of the partition nemesis (ms_set_nemesis, DESIGN.md 2.13): a cluster's op draws,
// delays and targets, and the rank-and-split of its servers into the two sides of a grudge.  One header for the
// kernel (k_nemesis in csrc/ms_kernels.cu) and the host (ms_set_nemesis's first instants, ms_nemesis_grudge), so
// that a caller turning a history record into sides computes exactly what the device did; the tests restate it
// independently in Python.
#pragma once
#include <stdint.h>
#include "ms_device.cuh"

namespace msd {

constexpr uint32_t kNemDrawKey = 0x4E454D00u;   // Philox(j, c, .., 0): op j of cluster c
constexpr uint32_t kNemRankKey = 0x4E454D01u;   // Philox(j, s, .., 0): server s's key in start op j
constexpr uint32_t kNemMaxGroup = 8192;
constexpr int64_t  kNemDefaultIntervalNs = 10000000000ll;   // --nemesis-interval 10 (core.clj:206-217)
constexpr int64_t  kNemMaxIntervalNs = 1ll << 50;           // keeps t_j + 2 interval far from overflow

// Per-cluster state in HBM: the instant of the next op (t_j), its index j, and the MS_HF_NEM_* code of the start
// that holds (0 = healthy): a stop clears what that start wrote, `comp` entries or the block of the pair matrix.
struct NemDev {
  int64_t  t;
  uint32_t op, part;
};

MS_HD void nem_draw(uint32_t seed_lo, uint32_t seed_hi, uint32_t cluster, uint32_t op, uint32_t x[4]) {
  philox4x32_10(op, cluster, kNemDrawKey, 0u, seed_lo, seed_hi, x);
}

// gen/stagger's integer delay, (x0 * 2 interval) >> 32, rounded up to whole ticks
MS_HD int64_t nem_delay_ns(uint32_t x0, int64_t interval_ns) {
  const uint64_t d = (uint64_t)(((unsigned __int128)x0 * (unsigned __int128)(2 * (uint64_t)interval_ns)) >> 32);
  return (int64_t)((d + (uint64_t)kTickNs - 1) / (uint64_t)kTickNs * (uint64_t)kTickNs);
}

MS_HD int64_t nem_add(int64_t t, int64_t d) { return t > INT64_MAX - d ? INT64_MAX : t + d; }

// the instant at which the cluster next acts: its next op, else the final stop at the time limit, else never
MS_HD int64_t nem_pending(const NemDev& n, int64_t limit_ns) {
  return n.t < limit_ns ? n.t : (n.part ? limit_ns : INT64_MAX);
}

// ms_nemesis_config.targets: bits 0-2 the component targets, bit 3 primaries (refused: the Maelstrom db has none),
// bit 4 majorities-ring; 0 = the three component targets
constexpr uint32_t kNemComponentTargets = 7u;
constexpr uint32_t kNemRingTarget = 0x10u;
constexpr uint32_t kNemTargetBits = kNemComponentTargets | kNemRingTarget;

// target mask and word 1 of the draw -> MS_HF_NEM_ONE / _MAJORITY / _MINORITY_THIRD / _MAJORITIES_RING: the enabled
// target (x1 * n_enabled) >> 32 in that order
MS_HD uint32_t nem_target(uint32_t mask, uint32_t x1) {
  mask = mask ? (mask & kNemTargetBits) : kNemComponentTargets;
  const uint32_t n = (mask & 1u) + ((mask >> 1) & 1u) + ((mask >> 2) & 1u) + ((mask >> 4) & 1u);
  uint32_t k = (uint32_t)(((uint64_t)x1 * n) >> 32);
  for (uint32_t t = 0; t < 5; t++)
    if ((mask >> t) & 1u) {
      if (k == 0) return t == 4 ? (uint32_t)MS_HF_NEM_MAJORITIES_RING : MS_HF_NEM_ONE + t;
      k--;
    }
  return MS_HF_NEM_ONE;
}

// majorities-ring: the server at ring position p receives from the one at position q iff (q - p + h) mod g < m, with
// m = g/2 + 1 and h = m/2 -- the window of m consecutive positions starting at i, given to the node at i + h.  Every
// member hears m members (itself included), no two the same set for g >= 3; the cut is one-way when m is even
MS_HD bool nem_ring_hears(uint32_t p, uint32_t q, uint32_t g) {
  const uint32_t m = g / 2 + 1, h = m / 2;
  return (q + g - p + h) % g < m;
}

// servers on side A: ranks below this
MS_HD uint32_t nem_side_a(uint32_t target, uint32_t g) {
  if (target == MS_HF_NEM_MAJORITY) return g / 2 + 1;
  if (target == MS_HF_NEM_MINORITY_THIRD) return g / 3 > 1 ? g / 3 : 1u;
  return 1u;
}

MS_HD uint32_t nem_key(uint32_t seed_lo, uint32_t seed_hi, uint32_t op, uint32_t server) {
  uint32_t x[4];
  philox4x32_10(op, server, kNemRankKey, 0u, seed_lo, seed_hi, x);
  return x[0];
}

// rank of member i among keys[0 .. g) in (key, index) order: a uniform shuffle of the cluster
MS_HD uint32_t nem_rank(const uint32_t* keys, uint32_t g, uint32_t i) {
  const uint32_t ki = keys[i];
  uint32_t r = 0;
  for (uint32_t k = 0; k < g; k++) r += (keys[k] < ki || (keys[k] == ki && k < i)) ? 1u : 0u;
  return r;
}

}  // namespace msd
