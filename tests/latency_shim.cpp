// Host shim over deepmimic_b200/csrc/kernels/dm_latency.cuh for tests/test_latency_cpu.py: the per-environment delay draw that
// dm_latency_reset_kernel runs on the device, compiled here with g++ so it can be checked against tests/latency_ref.py on the CPU.
#include "../deepmimic_b200/csrc/kernels/dm_latency.cuh"

using namespace dmk;

extern "C" {
int shim_lat_draw(int lo, int hi, unsigned long long seed, unsigned long long env, int resets) { return lat_draw(lo, hi, seed, env, resets); }
unsigned long long shim_lat_seed_key() { return kLatSeedKey; }
int shim_lat_bytes() { return static_cast<int>(sizeof(DevLat)); }
}
