// CPU checker of the distractor bodies: distractor_core.h compiled for the host in float64 (test infrastructure, like the oracle; the
// library itself has no CPU path).  Loaded by tests/test_distractors_*.py.
#include <string.h>
#include <vector>
#include "distractor_core.h"

extern "C" {

// scene[13] = table_z, txmin, txmax, tymin, tymax, button x, y, z, stack_top, stack_r, disc_r, disc0, disc1 (absolute disc z range);
// dt, iters, margin as the library uses them; gravity 10
static void scene_from(const double* sc, double dt, int iters, double margin, DcScene<double>& S) {
    S.table_z = sc[0]; S.txmin = sc[1]; S.txmax = sc[2]; S.tymin = sc[3]; S.tymax = sc[4];
    S.bx = sc[5]; S.by = sc[6]; S.bz = sc[7]; S.stack_top = sc[8]; S.stack_r = sc[9]; S.disc_r = sc[10]; S.disc0 = sc[11]; S.disc1 = sc[12];
    S.dt = dt; S.iters = iters; S.margin = margin; S.g = 10.0;
}

// Bodies B (f64[11][16], distractor_core.h layout) advanced by n_steps micro-steps against a fixed arm (narm spheres, f64[narm][4]);
// `kick` (nullable, impulse) is applied in micro-step `kick_step`.  traj (nullable): f64[n_steps][11][16] after every micro-step.
// touch (nullable): u32[2].  Returns 0, or 1 for a bad blob.
int dref_run(const double* blob, size_t bytes, const double* scene, double dt, int iters, double margin, double* B, const double* arm, int narm,
             int n_steps, const double* kick, int kick_step, double* traj, uint32_t* touch) {
    if (dc_blob_error(blob, bytes)) return 1;
    DcAssets<double> A; dc_assets_from_blob(blob, A);
    DcScene<double> S; scene_from(scene, dt, iters, margin, S);
    std::vector<DcRow<double>> rows(3 * DC_MAXC);
    DcTouch t = {0u, 0u};
    for (int s = 0; s < n_steps; ++s) {
        dc_step(A, S, B, arm, narm, (kick && s == kick_step) ? kick : nullptr, rows.data(), &t);
        if (traj) memcpy(traj + (size_t)s * DC_NBODY * DC_B_WORDS, B, sizeof(double) * DC_NBODY * DC_B_WORDS);
    }
    if (touch) { touch[0] = t.body; touch[1] = t.arm; }
    return 0;
}

// dref_run with a scene that changes per micro-step, as the kernel replays a trace: arm = f64[n_steps][narm][4], disc (nullable) =
// f64[n_steps][2] the disc's absolute z range, kicks (nullable) = f64[n_steps][3] impulses, applied where kick_on[s] != 0.
// touch (nullable): u32[2], OR-ed into.
int dref_run_steps(const double* blob, size_t bytes, const double* scene, double dt, int iters, double margin, double* B, const double* arm, int narm,
                   int n_steps, const double* disc, const double* kicks, const uint8_t* kick_on, double* traj, uint32_t* touch) {
    if (dc_blob_error(blob, bytes)) return 1;
    DcAssets<double> A; dc_assets_from_blob(blob, A);
    DcScene<double> S; scene_from(scene, dt, iters, margin, S);
    std::vector<DcRow<double>> rows(3 * DC_MAXC);
    DcTouch t = {0u, 0u};
    for (int s = 0; s < n_steps; ++s) {
        if (disc) { S.disc0 = disc[2 * s]; S.disc1 = disc[2 * s + 1]; }
        dc_step(A, S, B, arm + (size_t)s * narm * 4, narm, (kicks && kick_on[s]) ? kicks + 3 * s : nullptr, rows.data(), &t);
        if (traj) memcpy(traj + (size_t)s * DC_NBODY * DC_B_WORDS, B, sizeof(double) * DC_NBODY * DC_B_WORDS);
    }
    if (touch) { touch[0] |= t.body; touch[1] |= t.arm; }
    return 0;
}

// the islands of an adjacency (adj[k] bit m > k: bodies k and m are within the margin): root[k] = lowest slot of body k's island
void dref_island_roots(const uint32_t* adj, int* root) { dc_island_roots(adj, root); }

// reset()'s placement rule: B from 20 placement values (x0, y0, ..., x9, y9), 10 types and the button position
void dref_place(const double* xy, const int* type, double btn_x, double btn_y, double* B) { dc_place(B, xy, type, btn_x, btn_y); }

// the impulse of the kick for two normal draws
void dref_kick(double n0, double n1, double dt, double* imp) { dc_kick(n0, n1, dt, imp); }

}
