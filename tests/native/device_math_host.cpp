// Host build of the engine's pure device helpers (maelstrom_b200/csrc/ms_device.cuh is written
// with __host__ __device__ functions): lets the CPU test-suite pin the PRODUCT's Philox, fixed-point
// exponential, latency and shard-ownership code to the oracle and to the published vectors without
// a GPU.  Built by tests/test_device_math_host.py with g++.
struct uint4 { unsigned int x, y, z, w; };   // CUDA vector type, only named in pointer members of Params
#include "../../maelstrom_b200/csrc/ms_device.cuh"

extern "C" {
void dm_philox(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
  msd::philox4x32_10(ctr[0], ctr[1], ctr[2], ctr[3], key[0], key[1], out);
}
uint64_t dm_neg_log2_q32(uint64_t x) { return msd::neg_log2_q32(x); }
uint64_t dm_latency(uint32_t dist, uint32_t mean_ms, uint32_t scale, uint64_t exp_coeff, const uint32_t x[4]) {
  msd::NetParams np;
  np.loss_thresh = 0; np.exp_coeff = exp_coeff; np.dist = dist; np.mean_ms = mean_ms; np.scale = scale;
  np.pair_active = 0; np.comp_active = 0; np.any_removed = 0;
  return msd::latency_ms(np, x);
}
uint32_t dm_owner(uint32_t e, uint32_t n_servers, uint32_t g) { return msd::owner_of(e, n_servers, g); }
uint64_t dm_compact_round(uint64_t round, uint32_t round_lo) { return msd::compact_round(round, round_lo); }
uint32_t dm_sizeof_devstate(void) { return (uint32_t)sizeof(msd::DevState); }
uint32_t dm_sizeof_roundmeta(void) { return (uint32_t)sizeof(msd::RoundMeta); }
}
