// dm_course_kernel: the goal courses of the heading and target scenes (dm_course.cuh), one thread per environment.  capi.cu launches it only on
// handles with a course table (dm_set_goal_course): after dm_task_reset_kernel in dm_reset_clips, after the step launch of dm_update, and from
// the setter itself.
#include "dm_model.cuh"

namespace dmk {

// mode kCourseReset: environments whose reset counter moved start their course; kCourseStep: every course environment records, advances and
// writes its goal; kCourseStartAll: every course environment starts its course now (dm_set_goal_course).  Environments with n = 0 are untouched.
__global__ void dm_course_kernel(const DevModel* __restrict__ gm, DevState st, DevCourse* __restrict__ course, float* __restrict__ record, int num_real_envs,
                                 int mode) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= num_real_envs) return;
    DevCourse& c = course[env];
    if (c.n == 0) return;
    const DevModel& M = *gm;
    const int resets = st.flags[static_cast<size_t>(env) * kFlagInts + kFResets];
    if (mode == kCourseReset && resets == c.resets) return;
    double* tk = st.task + static_cast<size_t>(env) * kTaskDoubles;
    const float* sim = st.sim + static_cast<size_t>(env) * sim_stride(M.nl);
    const double rx = static_cast<double>(sim[0]) / M.scale, rz = static_cast<double>(sim[2]) / M.scale;
    const double tau = st.time[static_cast<size_t>(env) * kTimeDoubles + kTTimer];
    const int kind = task_base_kind(M.task_kind);
    float* rec = record + static_cast<size_t>(env) * kCourseRecordFloats;
    if (mode == kCourseStep) course_step(kind, M.task, c, tk, rx, rz, tau, rec);
    else course_start(kind, c, tk, rx, rz, tau, resets, rec);
}

}  // namespace dmk
