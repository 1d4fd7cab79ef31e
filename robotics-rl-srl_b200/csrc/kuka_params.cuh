// Kernel-parameter block of the Kuka kernels (float32 model + scene + env configuration).
//
// Passed BY VALUE as a __grid_constant__ kernel parameter: it lives in the constant bank, every
// access is warp-uniform, and ptxas folds the values into FFMA/FADD operands (c[0x0][...]) -- no load
// instructions and no registers for the robot model.  This replaces the per-reset asset loading of the
// reference (environments/kuka_gym/kuka.py:60-71, kuka_button_gym_env.py:221-239).
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include "kuka_model.h"

#define KK_NB 12           // movable bodies: PyBullet joints 0-8, 10, 11, 13
#define KK_ND 13           // + button glider
#define KK_MAXC 4          // contact rows kept per step (KM_SC_MAX_CONTACTS)
// one stored constraint row (contact normal / friction): J[14] at 0, 1 / D, target, W[14] at 16 -- 16-byte groups (eight 128-bit loads per row)
#define KK_ROW_J 0
#define KK_ROW_INVD 14
#define KK_ROW_TGT 15
#define KK_ROW_W 16
#define KK_ROWW 32

struct KukaParams {
    // ---- per body ----
    float org[KK_NB][3];   // joint origin in the parent frame
    float rot[KK_NB][9];   // parent <- child rotation at q = 0, row-major
    float axis[KK_NB][3];  // joint axis, child frame
    float mass[KK_NB];
    float com[KK_NB][3];
    float Ic[KK_NB][6];    // xx xy xz yy yz zz about the COM, body axes
    float damping[KK_NB];
    float lower[KK_NB], upper[KK_NB];
    float kp_dt[KK_NB];    // positionGain / dt
    float kd[KK_NB];
    float maxvel[KK_NB];   // <= 0: no clamp
    float maximp[KK_NB];   // force * dt
    int   tmode[KK_NB];    // 0: IK solution, others: 0 (end_effector_angle, finger_angle are identically 0)
    // saturating PGS sweep (kuka_device.cuh, "the SCALED system"): sigma_i = 2 maximp_i and the products the scaled problem needs
    float sat_sig[KK_NB], sat_isig[KK_NB], sat_isig2[KK_NB];
    float sat_ss[KK_NB * (KK_NB + 1) / 2], sat_iss[KK_NB * (KK_NB + 1) / 2];   // sigma_i sigma_j and its reciprocal, (i, j <= i) packed
    // ---- collision spheres ----
    int   nsph;
    int   sph_body[KM_MAX_SPHERES];
    float sph_c[KM_MAX_SPHERES][3];
    float sph_r[KM_MAX_SPHERES];
    int   sph_min_body;    // lowest body index that carries a sphere
    float sph_reach;       // max over spheres of |centre| + radius: no sphere surface is further from its body origin
    // ---- scene ----
    float base[3];
    float gz, dt, inv_dt;
    int   iters;
    float table_z, txmin, txmax, tymin, tymax;
    float btn_base[3];     // default button base origin
    float glider_z, gl_lo, gl_hi, btn_minv;
    float disc_r, disc_z0, disc_z1, stack_r, stack_top;
    float cdist, mu, erp, kl, ka;
    float ee_init[3];
    float box[6];          // active workspace box (small unless random_target): minx maxx miny maxy minz maxz
    float ikq[4];          // IK target orientation x y z w
    double ik_damp;
    int   ee_body, grip_body;
    float target_h, rand_x, rand_y;
    float btn_idle_imp, btn_kp_dt, btn_kd, btn_target, btn_maximp, lim_maximp, lim_eps;
    int   max_contacts;
    // ---- post-settle snapshot (state after the 500 zero-action steps of reset(), :242-247) ----
    float snap_q[KK_NB], snap_qd[KK_NB], snap_ee[3], snap_qb, snap_qdb;
    // ---- env configuration ----
    int   is_discrete, random_target, force_down, shape_reward, action_repeat, max_steps, auto_reset;
    int   action_joints;   // joint-space actions: use_inverse_kinematics = False (kuka_button_gym_env.py:238, kuka.py:158-161)
    float qinit[7];        // initial arm joint vector (kuka.py:65-66): what joint-space set-points are relative to
    int   two_buttons;     // Kuka2ButtonGymEnv: second button body, goal bookkeeping, IK damping 0.5 (kuka_2button_gym_env.py)
    float two_tgt_z;       // Z_TABLE + BUTTON_DISTANCE_HEIGHT: the z of both two-button targets
    int   moving_button;   // KukaMovingButtonGymEnv: the button slides along y (kuka_moving_button_gym_env.py:109-119)
    float max_distance;
    uint64_t seed, env_offset;
};

// Host side: the part of the parameter block that depends only on the model blob and the time step (dt <= 0: the blob's own) -- bodies,
// motors, the saturating sweep's products, collision spheres and scene constants.  The env configuration, solver iterations, workspace
// box, two-button overrides and RNG keys are the caller's (kuka_kernels.cu fill_params).  Returns an error message, or nullptr.
// Shared with the host check of the four-lane phases (tests/host/coop_host_check.cpp), so both run on the same model.
inline const char* kuka_params_from_blob(const double* d, size_t bytes, double dt, KukaParams& P) {
    if (!d || bytes < KM_HEADER_SIZE * sizeof(double) || d[KM_H_MAGIC] != KM_MAGIC || d[KM_H_VERSION] != KM_VERSION)
        return "kuka: bad model blob (magic/version)";
    if ((size_t)d[KM_H_TOTAL] * sizeof(double) != bytes || (int)d[KM_H_NBODY] != KK_NB || (int)d[KM_H_NSPHERE] > KM_MAX_SPHERES)
        return "kuka: bad model blob (size / body count / sphere count)";
    memset(&P, 0, sizeof(P));
    const double* sc = d + (int)d[KM_H_SCENE_OFF];
    if (!(dt > 0.0)) dt = sc[KM_SC_TIMESTEP];
    static const int parent[KK_NB] = {-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 7, 10};
    for (int i = 0; i < KK_NB; ++i) {
        const double* r = d + (int)d[KM_H_BODY_OFF] + i * KM_BODY_STRIDE;
        const double* c = d + (int)d[KM_H_CTRL_OFF] + i * KM_CTRL_STRIDE;
        if ((int)r[KM_B_PARENT] != parent[i] || (int)r[KM_B_JTYPE] != 0)
            return "kuka: the kernels are specialised for the 8-chain + two 2-link fingers revolute topology";
        for (int a = 0; a < 3; ++a) { P.org[i][a] = (float)r[KM_B_ORIGIN + a]; P.axis[i][a] = (float)r[KM_B_AXIS + a]; P.com[i][a] = (float)r[KM_B_COM + a]; }
        for (int a = 0; a < 9; ++a) P.rot[i][a] = (float)r[KM_B_ROT + a];
        for (int a = 0; a < 6; ++a) P.Ic[i][a] = (float)r[KM_B_INERTIA + a];
        P.mass[i] = (float)r[KM_B_MASS]; P.damping[i] = (float)r[KM_B_DAMPING];
        P.lower[i] = (float)r[KM_B_LOWER]; P.upper[i] = (float)r[KM_B_UPPER];
        P.kp_dt[i] = (float)(c[KM_C_KP] / dt); P.kd[i] = (float)c[KM_C_KD];
        P.maxvel[i] = (float)c[KM_C_MAXVEL]; P.maximp[i] = (float)(c[KM_C_MAXFORCE] * dt);
        P.tmode[i] = (int)c[KM_C_TARGET];
        P.snap_q[i] = (float)r[KM_B_QINIT];
    }
    for (int i = 0; i < KK_NB; ++i) {
        if (!(P.maximp[i] > 0.f)) return "kuka: every motor needs a positive force bound (the sweep carries impulses scaled to it)";
        const double sg = 2.0 * (double)P.maximp[i];
        P.sat_sig[i] = (float)sg; P.sat_isig[i] = (float)(1.0 / sg); P.sat_isig2[i] = (float)(1.0 / (sg * sg));
        for (int j = 0; j <= i; ++j) {
            const double ss = sg * 2.0 * (double)P.maximp[j];
            P.sat_ss[i * (i + 1) / 2 + j] = (float)ss; P.sat_iss[i * (i + 1) / 2 + j] = (float)(1.0 / ss);
        }
    }
    P.nsph = (int)d[KM_H_NSPHERE];
    P.sph_min_body = KK_NB; P.sph_reach = 0.f;
    for (int k = 0; k < P.nsph; ++k) {
        const double* sp = d + (int)d[KM_H_SPHERE_OFF] + k * KM_SPHERE_STRIDE;
        P.sph_body[k] = (int)sp[KM_S_BODY]; P.sph_r[k] = (float)sp[KM_S_RADIUS];
        for (int a = 0; a < 3; ++a) P.sph_c[k][a] = (float)sp[KM_S_CENTER + a];
        if (P.sph_body[k] < P.sph_min_body) P.sph_min_body = P.sph_body[k];
        const float reach = sqrtf(P.sph_c[k][0] * P.sph_c[k][0] + P.sph_c[k][1] * P.sph_c[k][1] + P.sph_c[k][2] * P.sph_c[k][2]) + P.sph_r[k];
        if (reach > P.sph_reach) P.sph_reach = reach * 1.0001f;
    }
    for (int a = 0; a < 3; ++a) { P.base[a] = (float)sc[KM_SC_BASE_POS + a]; P.btn_base[a] = (float)sc[KM_SC_BUTTON_BASE + a]; P.ee_init[a] = (float)sc[KM_SC_EE_INIT + a]; }
    P.gz = (float)sc[KM_SC_GRAVITY_Z]; P.dt = (float)dt; P.inv_dt = (float)(1.0 / dt);
    P.table_z = (float)sc[KM_SC_TABLE_TOP_Z]; P.txmin = (float)sc[KM_SC_TABLE_XMIN]; P.txmax = (float)sc[KM_SC_TABLE_XMAX];
    P.tymin = (float)sc[KM_SC_TABLE_YMIN]; P.tymax = (float)sc[KM_SC_TABLE_YMAX];
    P.glider_z = (float)sc[KM_SC_GLIDER_Z]; P.gl_lo = (float)sc[KM_SC_GLIDER_LOWER]; P.gl_hi = (float)sc[KM_SC_GLIDER_UPPER];
    P.btn_minv = (float)(1.0 / sc[KM_SC_BUTTON_MASS]);
    P.disc_r = (float)sc[KM_SC_DISC_RADIUS]; P.disc_z0 = (float)sc[KM_SC_DISC_Z0]; P.disc_z1 = (float)sc[KM_SC_DISC_Z1];
    P.stack_r = (float)sc[KM_SC_STACK_RADIUS]; P.stack_top = (float)sc[KM_SC_STACK_TOP];
    P.cdist = (float)sc[KM_SC_CONTACT_DIST]; P.mu = (float)sc[KM_SC_FRICTION]; P.erp = (float)sc[KM_SC_ERP];
    P.kl = (float)sc[KM_SC_LIN_DAMPING]; P.ka = (float)sc[KM_SC_ANG_DAMPING];
    for (int a = 0; a < 4; ++a) P.ikq[a] = (float)sc[KM_SC_IK_QUAT + a];
    P.ik_damp = sc[KM_SC_IK_DAMPING];
    P.ee_body = (int)sc[KM_SC_EE_BODY]; P.grip_body = (int)sc[KM_SC_GRIPPER_BODY];
    if (P.ee_body != 6 || P.grip_body != 8) return "kuka: kernels assume IK link 6 and gripper link 8 (kuka.py:31-32)";
    P.target_h = (float)sc[KM_SC_TARGET_HEIGHT]; P.rand_x = (float)sc[KM_SC_RAND_X]; P.rand_y = (float)sc[KM_SC_RAND_Y];
    P.btn_idle_imp = (float)sc[KM_SC_BTN_IDLE_IMPULSE]; P.btn_kp_dt = (float)(sc[KM_SC_BTN_KP] / dt); P.btn_kd = (float)sc[KM_SC_BTN_KD];
    P.btn_target = (float)sc[KM_SC_BTN_TARGET]; P.btn_maximp = (float)(sc[KM_SC_BTN_MAXFORCE] * dt);
    P.lim_maximp = (float)sc[KM_SC_LIMIT_MAX_IMPULSE]; P.lim_eps = (float)sc[KM_SC_LIMIT_EPS];
    P.max_contacts = (int)sc[KM_SC_MAX_CONTACTS];
    if (P.max_contacts > KK_MAXC) P.max_contacts = KK_MAXC;
    P.two_tgt_z = (float)(-0.2 + sc[KM_SC_TARGET_HEIGHT]);   // Z_TABLE + BUTTON_DISTANCE_HEIGHT (kuka_button_gym_env.py:26,35)
    for (int j = 0; j < 7; ++j) P.qinit[j] = P.snap_q[j];    // snap_q holds the initial joint vector until the settle steps have run
    return nullptr;
}
