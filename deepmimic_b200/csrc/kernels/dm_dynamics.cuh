// Per-environment dynamics: the factor table the step kernel's dynamics instantiation (dm_step_dyn_kernel) and the observation kernel's
// (dm_observe_dyn_kernel) read, and the randomisation rule that draws it at every reset (dm_set_dynamics_randomization).  Host / device-shared
// code like dm_push.cuh, driven on the host by tests/dynamics_shim.cpp and checked there against a Python restatement (tests/dynamics_ref.py).
//
// An environment with factors steps as the model built from edited asset files would: every PD controller's Kp and Kd times kp and kd, every
// joint's torque limit times torque_limit, every body's mass times its mass factor (both inertia tensors follow, since they are mass times a
// shape term), the contact friction coefficient times friction.  A fixed leaf lumped into its parent's composite body (humanoid3d's wrists)
// carries its parent's factor.  All factors 1 is the plain model.
//
// The draw: factor j of environment e in the episode with reset counter r is lo_j + u (hi_j - lo_j), u = task_u01(seed ^ "dynamics", global
// env id, 64 r + j), j = 0..3 friction, kp, kd, torque_limit, j = 4 + l the mass factor of link l (a lumped leaf copies its parent's instead).
// The product is rounded on its own (push_lerp), computed in double, stored as float.  A pure function of the seed, the global id and the reset
// counter: the same factors at any GPU count, and nothing to save beyond the rule.
#pragma once
#include "dm_push.cuh"

namespace dmk {

constexpr int kDynKinds = 5;   // friction, kp, kd, torque_limit, mass
enum DynSlot { kDFriction = 0, kDKp = 1, kDKd = 2, kDTlim = 3, kDMass = 4 /* + link */, kDTotalMass = 4 + 32, kDynFloats = 40 };

// One environment's entry of the table (indexed by environment id, not tile slot: placement by contact load moves it with its environment).
// total_mass is sum_l mass_l * factor_l, the denominator of every centre of mass; it equals DevModel::total_mass at unit factors.
struct DevDyn {
    float f[kDynFloats];
};
static_assert(sizeof(DevDyn) == 160, "DevDyn: 4 + 32 link factors + the total mass, padded to 16 bytes");

// the randomisation (a kernel parameter): [lo, hi] per kind, the draw stream, and the character's part of the rule
struct DynRand {
    double lohi[2 * kDynKinds];          // friction, kp, kd, torque_limit, mass
    unsigned long long seed, env_base;   // draw stream: task_u01(seed, env_base + env, 64 r + j)
    int nl, pad_;
    int leaf_parent[32];                 // the parent of a lumped fixed leaf, -1 for every other link
    float link_mass[32];                 // the character's masses (0 for a link without a shape, as the reference's total mass counts them)
};
// the draw stream's seed: the handle's seed with "dynamics", apart from the reset, task, push and expert-clip streams
constexpr unsigned long long kDynSeedKey = 0x64796e616d696373ull;
constexpr int kDynDrawsPerReset = 64;

// sum_l mass_l * factor_l in double, each product rounded on its own, in link order (the order of CharModel::total_mass)
DM_HD float dyn_total_mass(const float* link_mass, int nl, const float* f) {
    double m = 0.0;
    for (int l = 0; l < nl; ++l) m += push_mul(static_cast<double>(link_mass[l]), static_cast<double>(f[kDMass + l]));
    return static_cast<float>(m);
}

// one environment's factors for the episode with reset counter `resets` (env: its global id)
DM_HD void dyn_draw_env(const DynRand& R, unsigned long long env, int resets, DevDyn& d) {
    const unsigned long long k0 = static_cast<unsigned long long>(kDynDrawsPerReset) * static_cast<unsigned long long>(resets);
    for (int j = 0; j < 4; ++j) d.f[j] = static_cast<float>(push_lerp(R.lohi + 2 * j, task_u01(R.seed, env, k0 + j)));
    for (int l = 0; l < 32; ++l) d.f[kDMass + l] = 1.f;
    for (int l = 0; l < R.nl; ++l)
        if (R.leaf_parent[l] < 0) d.f[kDMass + l] = static_cast<float>(push_lerp(R.lohi + 8, task_u01(R.seed, env, k0 + 4 + l)));
    for (int l = 0; l < R.nl; ++l)
        if (R.leaf_parent[l] >= 0) d.f[kDMass + l] = d.f[kDMass + R.leaf_parent[l]];
    d.f[kDTotalMass] = dyn_total_mass(R.link_mass, R.nl, d.f);
    for (int k = kDTotalMass + 1; k < kDynFloats; ++k) d.f[k] = 0.f;
}

}  // namespace dmk
