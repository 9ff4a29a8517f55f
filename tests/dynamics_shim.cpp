// Host shim over deepmimic_b200/csrc/kernels/dm_dynamics.cuh for tests/test_dynamics_cpu.py: the per-environment dynamics draw that
// dm_dyn_draw_kernel runs on the device, compiled here with g++ so it can be checked against tests/dynamics_ref.py on the CPU.
#include "../deepmimic_b200/csrc/kernels/dm_dynamics.cuh"

#include <cstring>

using namespace dmk;

extern "C" {
// lohi [10]; leaf_parent, link_mass [nl]; out: the environment's DevDyn entry (kDynFloats floats)
void shim_dyn_draw(const double* lohi, unsigned long long seed, unsigned long long env, int resets, int nl, const int* leaf_parent, const float* link_mass,
                   float* out) {
    DynRand R;
    std::memset(&R, 0, sizeof(R));
    for (int k = 0; k < 2 * kDynKinds; ++k) R.lohi[k] = lohi[k];
    R.seed = seed; R.env_base = 0; R.nl = nl;
    for (int l = 0; l < 32; ++l) { R.leaf_parent[l] = l < nl ? leaf_parent[l] : -1; R.link_mass[l] = l < nl ? link_mass[l] : 0.f; }
    DevDyn d;
    dyn_draw_env(R, env, resets, d);
    std::memcpy(out, d.f, sizeof(d.f));
}
int shim_dyn_floats() { return kDynFloats; }
unsigned long long shim_dyn_seed_key() { return kDynSeedKey; }
}
