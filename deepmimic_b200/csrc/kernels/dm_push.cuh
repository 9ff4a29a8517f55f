// Pushes: the push-table entry the step kernel applies, and the random push schedule that refills it during training rollouts
// (dm_set_push_schedule).  Host / device-shared code like dm_task.cuh, driven on the host by tests/push_schedule_shim.cpp and checked there
// against a Python restatement of the rule and the draw stream (tests/push_schedule_ref.py).
//
// The schedule is this library's own: the reference's random-perturbation option (cSceneSimChar) is not restated.  One thread per environment
// (dm_push_schedule_kernel, at the head of every dm_update of a scheduled handle) runs push_schedule_env on a real environment that is not
// frozen (done flag clear):
//   1. its reset counter moved since the block was last initialised: a new episode, k = 0, last_end = 0;
//   2. its entry is empty (body -1): five draws u = task_u01(seed, global env id, k++) in the order gap, body index, magnitude, direction angle,
//      duration; start = max(last_end + gap, t) with t the episode timer now (a start already passed is moved to t, never skipped); the force is
//      horizontal, (F cos a, 0, F sin a) with a in [0, 2 pi) (run.py: push_plan); last_end = start + duration.
// Every product is rounded on its own (no fused multiply-add on the device), so the device, g++ and the Python restatement agree bit for bit.
#pragma once
#include "dm_task.cuh"

namespace dmk {

// A timed external force on one body (dm_set_pushes, dm_set_push_schedule): force (world axes, unscaled N) at the body's COM in both Bullet
// sub-steps of every update whose timer value at its start t satisfies start <= t < start + duration.  body -1: none; the step kernel sets it at
// the commit of the update after which t >= start + duration, dm_reset at the environment's reset.  A handle's push table holds one entry per
// environment id (not tile slot, so placement by contact load moves a push with its environment) and reaches dm_step_push_kernel as its last
// parameter, not as a DevState field: a larger DevState would move every later parameter of every kernel that takes it.
struct DevPush {
    float force[3];
    int body;
    double start, duration;
};
static_assert(sizeof(DevPush) == 32, "DevPush: the step kernel reads force and body as one float4");

constexpr int kMaxPushBodies = 32;
// schedule parameters (a kernel parameter): bodies drawn from, and [lo, hi] of the magnitude (N), the duration (s) and the gap (s)
struct PushSchedule {
    int n_bodies, pad_;
    int bodies[kMaxPushBodies];
    double force[2], duration[2], gap[2];
    unsigned long long seed, env_base;   // draw stream: task_u01(seed, env_base + env, k)
};
// schedule block, doubles per environment
constexpr int kPushSchedDoubles = 3;
enum PushSchedSlot { kPResetSeen = 0, kPCounter = 1, kPLastEnd = 2 };
// the draw stream's seed: the handle's seed with "pushes", apart from the reset (seed), task (seed ^ "tasks") and expert-clip streams
constexpr unsigned long long kPushSeedKey = 0x707573686573ull;

DM_HD double push_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
DM_HD double push_lerp(const double* lohi, double u) { return lohi[0] + push_mul(u, lohi[1] - lohi[0]); }

// one environment's schedule step: resets = its reset counter, timer = its episode timer now, s = its schedule block, e = its push-table entry
DM_HD void push_schedule_env(const PushSchedule& P, unsigned long long env, int resets, double timer, double* s, DevPush& e) {
    if (static_cast<double>(resets) != s[kPResetSeen]) { s[kPResetSeen] = static_cast<double>(resets); s[kPCounter] = 0.0; s[kPLastEnd] = 0.0; }
    if (e.body != -1) return;
    const unsigned long long k = static_cast<unsigned long long>(s[kPCounter]);
    const double gap = push_lerp(P.gap, task_u01(P.seed, env, k));
    int i = static_cast<int>(push_mul(task_u01(P.seed, env, k + 1), static_cast<double>(P.n_bodies)));
    if (i > P.n_bodies - 1) i = P.n_bodies - 1;
    const double mag = push_lerp(P.force, task_u01(P.seed, env, k + 2));
    const double ang = push_mul(2.0 * 3.14159265358979323846, task_u01(P.seed, env, k + 3));
    const double dur = push_lerp(P.duration, task_u01(P.seed, env, k + 4));
    s[kPCounter] = static_cast<double>(k + 5);
    const double start = fmax(s[kPLastEnd] + gap, timer);
    e.force[0] = static_cast<float>(push_mul(mag, cos(ang))); e.force[1] = 0.f; e.force[2] = static_cast<float>(push_mul(mag, sin(ang)));
    e.body = P.bodies[i]; e.start = start; e.duration = dur;
    s[kPLastEnd] = start + dur;
}

}  // namespace dmk
