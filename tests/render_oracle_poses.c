/* World poses of every body of an oracle env, from the fp64 oracle's own forward kinematics (the static kinematics() of
 * oracle/rexsim_oracle.c, compiled into this unit unchanged).  Used by tests/render_oracle.py only. */
#include "../oracle/rexsim_oracle.c"

/* R: [nb][9] body -> world rotation (row-major), p: [nb][3] body origin in the world */
void rexo_link_poses(const RexoSim* s, int i, double* R, double* p) {
    static Scratch k;
    kinematics(s, &s->env[i], &k);
    for (int b = 0; b < s->m.nb; b++) {
        for (int a = 0; a < 9; a++) R[9 * b + a] = (double)k.Rw[b][a];
        for (int a = 0; a < 3; a++) p[3 * b + a] = (double)k.pw[b][a];
    }
}
