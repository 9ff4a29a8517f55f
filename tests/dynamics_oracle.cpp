// The CPU oracle with another contact friction coefficient, for tests/test_dynamics_gpu.py: oracle/dm_oracle.cpp as it is, plus one entry
// that sets the coefficient Bullet's solver uses for every contact (the reference's link friction times the ground's).  Masses, gains and
// torque limits need no entry: the test edits them in a copy of the asset files.
#include "../oracle/dm_oracle.cpp"

extern "C" {
void dmo_set_friction(void* h, double mu) { static_cast<orc::Oracle*>(h)->friction = mu; }
}
