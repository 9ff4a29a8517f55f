// Host shim over deepmimic_b200/csrc/kernels/dm_push.cuh for tests/test_push_schedule_cpu.py: the per-environment push schedule that
// dm_push_schedule_kernel runs on the device, compiled here with g++ so it can be checked against tests/push_schedule_ref.py on the CPU.
#include "../deepmimic_b200/csrc/kernels/dm_push.cuh"

#include <cstring>

using namespace dmk;

extern "C" {
// bodies [n_bodies]; bounds: force lo, hi, duration lo, hi, gap lo, hi.  s: the environment's schedule block (kPushSchedDoubles); entry: body
// (int), force [3] (float), start and duration (double), read and written in place
void shim_push_schedule(const int* bodies, int n_bodies, const double* bounds, unsigned long long seed, unsigned long long env, int resets,
                        double timer, double* s, int* body, float* force, double* window) {
    PushSchedule P;
    std::memset(&P, 0, sizeof(P));
    P.n_bodies = n_bodies;
    for (int i = 0; i < n_bodies; ++i) P.bodies[i] = bodies[i];
    for (int k = 0; k < 2; ++k) { P.force[k] = bounds[k]; P.duration[k] = bounds[2 + k]; P.gap[k] = bounds[4 + k]; }
    P.seed = seed; P.env_base = 0;
    DevPush e;
    e.body = *body; e.force[0] = force[0]; e.force[1] = force[1]; e.force[2] = force[2]; e.start = window[0]; e.duration = window[1];
    push_schedule_env(P, env, resets, timer, s, e);
    *body = e.body; force[0] = e.force[0]; force[1] = e.force[1]; force[2] = e.force[2]; window[0] = e.start; window[1] = e.duration;
}
int shim_push_sched_doubles() { return kPushSchedDoubles; }
unsigned long long shim_push_seed_key() { return kPushSeedKey; }
}
