// Control latency: the per-environment table the step kernel's latency instantiation (dm_step_latency_kernel) reads, and the randomisation rule
// that draws its delays at every reset (dm_set_action_latency_randomization).  Host / device-shared code like dm_dynamics.cuh, driven on the
// host by tests/latency_shim.cpp and checked there against a Python restatement (tests/latency_ref.py).
//
// Environment e has a delay d_e, a whole number of updates in [0, updates_per_action - 1].  The PD targets of an action set by dm_set_action
// take effect at the Stable-PD stage of the (d_e + 1)-th update after it; until then the previous targets act.  One action at most is pending:
// dm_set_action_latency_kernel writes its targets into the entry (tg, the target slot's layout) with due = the environment's update counter
// (kFUpdates) + d_e, a later action replaces it, and the step kernel copies tg into the target slot at the update whose counter equals due.
// d_e = 0 writes the target slot at once, as the plain kernel does.  A reset drops the pending action and holds the reset pose
// (dm_latency_reset_kernel).
//
// The draw: the delay of environment e in the episode with reset counter r is lo + min(hi - lo, floor(u (hi - lo + 1))),
// u = task_u01(seed ^ "latency", global env id, r).  A pure function of the seed, the global id and the reset counter: the same delays at any
// GPU count, and nothing to save beyond the rule.
#pragma once
#include "dm_task.cuh"

namespace dmk {

// One environment's entry of the table (indexed by environment id, not tile slot: placement by contact load moves it with its environment).
struct DevLat {
    int delay;        // d_e, in updates
    int due;          // the update counter (kFUpdates) at whose Stable-PD stage tg takes effect; -1: no action pending
    int resets;       // the reset counter (kFResets) the entry last saw: a change is a reset (the hold and the draw)
    int pad_;
    float tg[4 * 32];   // the pending action's PD targets, one float4 per link in the target slot's layout (sim + 16 + 8 nl)
};
static_assert(sizeof(DevLat) == 528, "DevLat: four ints and 32 float4 targets");

// the randomisation (a kernel parameter): [lo, hi] in updates and the draw stream
struct LatRand {
    int lo, hi;
    unsigned long long seed, env_base;   // draw stream: task_u01(seed, env_base + env, r)
};
// the draw stream's seed: the handle's seed with "latency", apart from the reset, task, push, dynamics and expert-clip streams
constexpr unsigned long long kLatSeedKey = 0x6c6174656e6379ull;

// the delay of one environment (env: its global id) in the episode with reset counter `resets`
DM_HD int lat_draw(int lo, int hi, unsigned long long seed, unsigned long long env, int resets) {
    const double u = task_u01(seed, env, static_cast<unsigned long long>(resets));
    const int span = hi - lo;
    const int k = static_cast<int>(floor(u * static_cast<double>(span + 1)));
    return lo + (k < span ? k : span);
}

}  // namespace dmk
