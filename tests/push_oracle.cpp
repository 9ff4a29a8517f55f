// The CPU oracle with a timed push, for tests/test_push_*.py: oracle/dm_oracle.cpp as it is, plus one entry that applies an external force
// for one Update.  cWorld::Update keeps applied forces through stepSimulation until its final clearForces, and nothing in cSceneSimChar::Update
// before stepSimulation touches them, so the force is added to the body's link (Bullet's link frame sits at the body's COM) right before the
// oracle's own Update and acts in both of its sub-steps.
#include "../oracle/dm_oracle.cpp"

extern "C" {
// One Update(dt), with force (world axes, unscaled N) times the world scale on `body` when body >= 0 and the timer value at the update's start t
// satisfies start <= t < start + duration (the scale rule of gravity: the unscaled character sees F / m).
void dmo_push_update(void* h, double dt, int body, const double* force, double start, double duration) {
    orc::Oracle* o = static_cast<orc::Oracle*>(h);
    const double t = o->timer_time;
    if (body >= 0 && start <= t && t < start + duration)
        o->mb.links[body].appliedForce += orc::F3(static_cast<float>(force[0] * o->scale), static_cast<float>(force[1] * o->scale), static_cast<float>(force[2] * o->scale));
    o->Update(dt);
}
}
