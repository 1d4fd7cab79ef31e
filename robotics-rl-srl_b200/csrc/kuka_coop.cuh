// Kuka physics, once-per-micro-step part, FOUR LANES PER ENVIRONMENT (round 2).
//
// What runs once per micro-step -- forward kinematics, collision detection, inverse kinematics, CRBA + RNEA, Cholesky and M^-1 --
// was a small share of the warp instructions but a large share of the time of kuka_kernel in round 1: 100 KB of
// straight-line code streamed through the instruction caches by ONE warp per scheduler with 7 of 32 lanes alive, each instruction
// costing several cycles (instruction-fetch and scoreboard stalls).  Here an env is a GROUP of KC_G = 4 adjacent lanes:
//   * per-body work (12 bodies: local rotations, world inertias, spatial inertias, body wrenches, momentum vectors, rows of M, columns of
//     L^-1, entries of M^-1, collision spheres, contact rows) is dealt round-robin to the 4 lanes -- a third of the instructions per warp,
//   * the strictly sequential pieces (transform chain, tree prefix / suffix sums, Cholesky pivots) are split by matrix row or by scalar
//     component, or done redundantly where splitting would cost more than it saves (the 7x7 float64 IK solve),
//   * everything that crosses lanes goes through a per-env scratch area in SHARED memory and a __syncwarp() -- no thread-local arrays,
//     no 3.4 KB stack frame.
// All 4 lanes of a group carry identical copies of the env state and run the env logic and the PGS sweep redundantly (SIMT: free), so the
// control flow of the kernel stays uniform within a group.
//
// The header compiles for the host as well (tests/coop_host_check.cpp runs the 4 lanes of a group one after the other, phase by phase, and
// compares with the one-thread-per-env functions of kuka_device.cuh): every phase is a function of (scratch, lane) only.
#pragma once
#include <math.h>
#include <stdint.h>
#include "kuka_params.cuh"

#if defined(__CUDACC__)
#define KC_F __device__ __forceinline__
#else
#define KC_F inline
#endif
#if defined(__CUDA_ARCH__)
#define KC_RSQRT(x) rsqrtf(x)
#else
#define KC_RSQRT(x) (1.0f / sqrtf(x))
#endif

// Diagnostic build (scripts/build_variant.sh phases -DKK_PHASES, scripts/kuka_phase_timing.py): clock() accumulators per phase of the
// micro-step loop, in registers, stored per env slot at the end of the launch.  Separate from KK_TIMING, whose convergence probe adds
// instructions to every sweep row.  KK_PH(clk, k) charges the cycles since the previous mark to phase k; without KK_PHASES it is empty.
// 32-bit accumulators (a slot runs ~10^7 cycles per launch): half the registers of clock64() ones, so the 21 marks add fewer spills.
// The fast sweeps are charged to one of two phases, by the copy of the loop the warp ran (no lane
// watching a contact, or the watch copy); `nwatch` counts the physics steps of the slot that ran the watch copy.
enum {
    KK_PH_KIN_LOCAL = 0, KK_PH_KIN_CHAIN, KK_PH_KIN_BODY, KK_PH_KIN_COLLECT,              // kinematics + collision (kc_kinematics)
    KK_PH_IK_BUILD, KK_PH_IK_SOLVE,                                                     // J, error, J^T J, J^T e / the 7x7 solve
    KK_PH_DYN_D1, KK_PH_DYN_D2, KK_PH_DYN_D3, KK_PH_DYN_D4, KK_PH_DYN_D5, KK_PH_DYN_D6, KK_PH_DYN_D7,   // kc_dynamics (+ loading M, bias)
    KK_PH_CHOL,                                                                         // Cholesky + M^-1
    KK_PH_SETUP, KK_PH_ROWS, KK_PH_EULER,                                               // v0 + motor / limit set-up, contact rows + scaling, Euler
    KK_PH_FAST_QUIET, KK_PH_FAST_WATCH, KK_PH_GENERAL, KK_PH_ENV, KK_NPH
};
#if defined(KK_PHASES) && defined(__CUDACC__)
struct KkPhaseClock { unsigned last; unsigned acc[KK_NPH]; unsigned nwatch; };
#define KK_PH(clk, k) do { if (clk) { const unsigned t_ = (unsigned)clock(); (clk)->acc[k] += t_ - (clk)->last; (clk)->last = t_; } } while (0)
#else
struct KkPhaseClock { long long dummy; };
#define KK_PH(clk, k) do { (void)(clk); } while (0)
#endif

#define KC_G 4               // lanes per env
#define KC_BS 53             // per-body record stride in words (odd: 4 lanes on 4 different bodies hit 4 different banks)
#define KC_CS 25             // per-body constant record stride (odd)

// ---- per-body record (two fields of the kinematics are dead by the time the dynamics write theirs and share the storage) -----------
enum {
    KB_R = 0,     // [9] world rotation of the body frame         (chain -> body phase, IK)   | later N, F, PM
    KB_N = 0,     // [3] body wrench about the origin -> sub-tree sum
    KB_F = 3,     // [3]
    KB_PM = 6,    // [3] linear momentum of the composite under unit joint rate
    KB_P = 9,     // [3] joint frame origin, world
    KB_A = 12,    // [3] joint axis, world
    KB_PV = 15,   // [3] p x a
    KB_C = 18,    // [3] centre of mass, world
    KB_IW = 21,   // [6] rotational inertia about the COM, world axes
    KB_M = 27,    // [1] mass                      -> composite mass of the sub-tree
    KB_H = 28,    // [3] m c                       -> composite first moment
    KB_IO = 31,   // [6] inertia about the origin  -> composite inertia
    KB_B = 37,    // [9] local rotation rot_i * Rodrigues(axis_i, q_i)   (phase 1 -> chain)   | later W, VO, AW
    KB_W = 37,    // [3] angular velocity            (prefix sum over the ancestors)
    KB_VO = 40,   // [3] velocity of the body-fixed point at the world origin
    KB_AW = 43,   // [3] per-body term, then angular acceleration (prefix sum)
    KB_AV = 46,   // [3] per-body term, then acceleration of the point at the origin (gravity as base acceleration)
    KB_LM = 49,   // [3] angular momentum about the origin
};
// ---- rest of the scratch map ----------------------------------------------------------------------------------------------------
#define KC_MS 13                                   // row stride of the 12 x 12 matrices (odd)
#define KC_OFF_LINK (KK_NB * KC_BS)                // [8] (6 unused), manifold flags, number of contact records
#define KC_OFF_CT (KC_OFF_LINK + 8)                // KK_MAXC contact records of KC_CTS words: body, shape, dist, n[3], pt[3]
#define KC_CTS 9
#define KC_OFF_MA (KC_OFF_CT + KK_MAXC * KC_CTS)   // M, lower triangle (every lane then inverts it in registers)
#define KC_OFF_BIAS (KC_OFF_MA + KK_NB * KC_MS)    // [12] bias torques
#define KC_OFF_ROWS (((KC_OFF_BIAS + KK_NB + 3) / 4) * 4)   // 3 * KK_MAXC constraint rows of KC_RS words in the KK_ROW_* layout (kuka_params.cuh), 16-byte aligned
#define KC_RS 36                                   // = 4 (mod 32): the 4 lanes that fill 4 consecutive rows hit different banks; a multiple of 4 words
#define KC_OFF_WT (KC_OFF_ROWS + 3 * KK_MAXC * KC_RS)   // watch matrix [12][4]: Wt[i][c] = W'_i of normal row c < nc, written and read by lane c of the group
#define KC_OFF_END (KC_OFF_WT + KK_NB * 4)
#define KC_OFF_CAND KC_OFF_MA                      // collision candidates per sphere (count, then KC_CANDS records of 8 words: shape, dist, n, pt):
#define KC_CANDS 3                                 // consumed by the collect phase before the dynamics write M, L, rows -- same storage
#define KC_CANDW (1 + KC_CANDS * 8)
#define KC_WORDS KC_OFF_END
#define KC_ROWS4 ((KC_WORDS + 3) / 4)              // 16-byte rows per env
static_assert(KC_BS % 4 == 1 && KC_MS % 4 == 1 && KC_CS % 4 == 1, "lane-indexed strides must be odd (1 or 3 mod 4)");
static_assert(KC_RS % 32 == 4 && KC_RS >= KK_ROWW && KC_OFF_ROWS % 4 == 0 && KC_OFF_WT % 4 == 0 && KK_MAXC == 4, "constraint rows: 16-byte aligned, consecutive rows 4 banks apart");
static_assert(KC_OFF_CAND + KM_MAX_SPHERES * KC_CANDW <= KC_OFF_END, "collision candidates must fit in the storage they share");

// per-CTA constant tables (same for every env): body records of KC_CS words, then sphere records of 5 words
enum { KCB_ORG = 0, KCB_ROT = 3, KCB_AXIS = 12, KCB_COM = 15, KCB_IC = 18, KCB_MASS = 24 };
#define KC_CONST_SPH (KK_NB * KC_CS)               // sphere s: body (as float), centre xyz, radius
#define KC_CONST_WORDS (KC_CONST_SPH + KM_MAX_SPHERES * 5)

// Scratch addressing: word w of the env in slot e (= 8 * warp + group) lives at  e * KC_ES + w.  KC_ES = 4 (mod 32), so the 8 groups of a warp
// start 4 banks apart; every stride a lane index is multiplied with (per-body records, matrix rows) is = 1 (mod 4), so the 4 lanes of a
// group working on 4 different bodies / rows stay in 4 different banks: the same field of 4 bodies in 7 groups = 28 distinct banks.
#define KC_ES (((KC_WORDS + 27) / 32) * 32 + 4)
struct KcScratch {
    float* b;          // word 0 of this env
    KC_F float& operator[](int w) const { return b[w]; }
};

KC_F void kc_fill_const(const KukaParams& P, float* tab, int tid, int nthreads) {
    for (int k = tid; k < KK_NB * KC_CS; k += nthreads) {
        const int i = k / KC_CS, f = k % KC_CS;
        float v;
        if (f < KCB_ROT) v = P.org[i][f];
        else if (f < KCB_AXIS) v = P.rot[i][f - KCB_ROT];
        else if (f < KCB_COM) v = P.axis[i][f - KCB_AXIS];
        else if (f < KCB_IC) v = P.com[i][f - KCB_COM];
        else if (f < KCB_MASS) v = P.Ic[i][f - KCB_IC];
        else v = P.mass[i];
        tab[k] = v;
    }
    for (int k = tid; k < KM_MAX_SPHERES * 5; k += nthreads) {
        const int s = k / 5, f = k % 5;
        tab[KC_CONST_SPH + k] = f == 0 ? (float)P.sph_body[s] : f < 4 ? P.sph_c[s][f - 1] : P.sph_r[s];
    }
}

// ---- small vector helpers with explicit fused operations (identical results on host and device) ------------------------------------
struct kc3 { float x, y, z; };
KC_F kc3 kc_mk(float x, float y, float z) { kc3 r; r.x = x; r.y = y; r.z = z; return r; }
KC_F kc3 kc_add(kc3 a, kc3 b) { return kc_mk(a.x + b.x, a.y + b.y, a.z + b.z); }
KC_F kc3 kc_sub(kc3 a, kc3 b) { return kc_mk(a.x - b.x, a.y - b.y, a.z - b.z); }
KC_F kc3 kc_scale(float s, kc3 a) { return kc_mk(s * a.x, s * a.y, s * a.z); }
KC_F kc3 kc_fma(float s, kc3 a, kc3 b) { return kc_mk(fmaf(s, a.x, b.x), fmaf(s, a.y, b.y), fmaf(s, a.z, b.z)); }   // s a + b
KC_F float kc_dot(kc3 a, kc3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
KC_F kc3 kc_cross(kc3 a, kc3 b) { return kc_mk(fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x))); }
KC_F kc3 kc_symv(const float* I, kc3 v) {
    return kc_mk(fmaf(I[2], v.z, fmaf(I[1], v.y, I[0] * v.x)), fmaf(I[4], v.z, fmaf(I[3], v.y, I[1] * v.x)), fmaf(I[5], v.z, fmaf(I[4], v.y, I[2] * v.x)));
}
template <class S> KC_F kc3 kc_ld3(const S& s, int w) { return kc_mk(s[w], s[w + 1], s[w + 2]); }
template <class S> KC_F void kc_st3(const S& s, int w, kc3 v) { s[w] = v.x; s[w + 1] = v.y; s[w + 2] = v.z; }
KC_F int kc_parent(int i) { return i == 0 ? -1 : i == 10 ? 7 : i - 1; }
// i ancestor-or-self of j  (chain 0..7 precedes everything; 8 -> 9; 10 -> 11)
KC_F bool kc_anc(int i, int j) { return (i == j) || (i <= 7 && i < j) || (i == 8 && j == 9) || (i == 10 && j == 11); }
// value k of a 12-vector held in registers by every lane, for the body u + 4 k of lane u (static register indices only)
#define KC_SEL4(arr, k, u) ((u) == 0 ? (arr)[4 * (k)] : (u) == 1 ? (arr)[4 * (k) + 1] : (u) == 2 ? (arr)[4 * (k) + 2] : (arr)[4 * (k) + 3])
// index of the lowest set bit of x != 0
KC_F int kc_lowest_bit(unsigned x) {
#if defined(__CUDA_ARCH__)
    return __ffs(x) - 1;
#else
    return __builtin_ctz(x);
#endif
}

// sphere vs upright finite cylinder (axis +z through (cx, cy), z in [z0, z1], radius R)
KC_F void kc_sphere_cylinder(kc3 s, float r, float cx, float cy, float z0, float z1, float R, float& dist, kc3& n) {
    const float dx = s.x - cx, dy = s.y - cy;
    const float rho = sqrtf(dx * dx + dy * dy);
    const kc3 radial = rho > 1e-12f ? kc_mk(dx / rho, dy / rho, 0.f) : kc_mk(1.f, 0.f, 0.f);
    float d;
    if (s.z >= z1 || s.z <= z0) {
        const float zf = s.z >= z1 ? z1 : z0;
        if (rho <= R) { d = fabsf(s.z - zf); n = kc_mk(0.f, 0.f, s.z >= z1 ? 1.f : -1.f); }
        else { const kc3 vec = kc_mk(dx - radial.x * R, dy - radial.y * R, s.z - zf); d = sqrtf(kc_dot(vec, vec)); n = kc_scale(1.0f / d, vec); }
    } else if (rho > R) {
        d = rho - R; n = radial;
    } else {
        const float d_top = z1 - s.z, d_side = R - rho;
        if (d_top <= d_side) { d = -d_top; n = kc_mk(0.f, 0.f, 1.f); } else { d = -d_side; n = radial; }
    }
    dist = d - r;
}

// What the kinematics phases need from the env state (identical in the 4 lanes of a group).
struct KcKinIn {
    float q[KK_NB];
    float qb, qb2;              // button gliders
    float bbx, bby, bbz;        // button base
    float bb2x, bb2y;           // second button base (two-button kind)
};

// ================================================================ kinematics ======================================================
// Phase 1: local rotations of the lane's bodies.
// The constant table and the scratch area are both shared memory: a table load that follows a scratch store in program order waits for
// it.  So every phase loads its constants (and the scratch words it reads) ahead of its stores.
template <class S>
KC_F void kc_ph_local(const S& s, const float* tab, const KcKinIn& in, int u) {
    float ax[KK_NB / KC_G][3], rot[KK_NB / KC_G][9];
#pragma unroll
    for (int k = 0; k < KK_NB / KC_G; ++k) {
        const float* c = tab + (u + KC_G * k) * KC_CS;
#pragma unroll
        for (int t = 0; t < 3; ++t) ax[k][t] = c[KCB_AXIS + t];
#pragma unroll
        for (int t = 0; t < 9; ++t) rot[k][t] = c[KCB_ROT + t];
    }
#pragma unroll
    for (int k = 0; k < KK_NB / KC_G; ++k) {
        const int i = u + KC_G * k;
        const float qi = KC_SEL4(in.q, k, u);
        float sn, cs;
        sincosf(qi, &sn, &cs);
        const float t = 1.f - cs, ax0 = ax[k][0], ay = ax[k][1], az = ax[k][2];
        const float Q[9] = {cs + t * ax0 * ax0, t * ax0 * ay - sn * az, t * ax0 * az + sn * ay,
                            t * ax0 * ay + sn * az, cs + t * ay * ay, t * ay * az - sn * ax0,
                            t * ax0 * az - sn * ay, t * ay * az + sn * ax0, cs + t * az * az};
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int cc = 0; cc < 3; ++cc)
                s[i * KC_BS + KB_B + 3 * r + cc] = fmaf(rot[k][3 * r + 2], Q[6 + cc], fmaf(rot[k][3 * r + 1], Q[3 + cc], rot[k][3 * r] * Q[cc]));
    }
}

// Phase 2: the transform chain, one ROW of every world rotation (and one component of every origin) per lane; lane 3 idles.  The local
// rotation and the origin offset of body i + 2 are loaded before the stores of body i (registers: static indices after unrolling).
template <class S>
KC_F void kc_ph_chain(const S& s, const float* tab, const KukaParams& P, int u) {
    if (u >= 3) return;
    float B[KK_NB][9], O[KK_NB][3];
#define KC_CHAIN_LOAD(j)                                                                  \
    {                                                                                     \
        _Pragma("unroll") for (int t = 0; t < 9; ++t) B[j][t] = s[(j) * KC_BS + KB_B + t]; \
        _Pragma("unroll") for (int t = 0; t < 3; ++t) O[j][t] = tab[(j) * KC_CS + KCB_ORG + t]; \
    }
    KC_CHAIN_LOAD(0)
    KC_CHAIN_LOAD(1)
    float R0 = u == 0 ? 1.f : 0.f, R1 = u == 1 ? 1.f : 0.f, R2 = u == 2 ? 1.f : 0.f;
    float p = u == 0 ? P.base[0] : u == 1 ? P.base[1] : P.base[2];
    float S0 = R0, S1 = R1, S2 = R2, sp = p;   // body 7: where the second finger restarts
#pragma unroll
    for (int i = 0; i < KK_NB; ++i) {
        if (i + 2 < KK_NB) KC_CHAIN_LOAD(i + 2)
        if (i == 10) { R0 = S0; R1 = S1; R2 = S2; p = sp; }
        p = fmaf(R2, O[i][2], fmaf(R1, O[i][1], fmaf(R0, O[i][0], p)));
        const float n0 = fmaf(R2, B[i][6], fmaf(R1, B[i][3], R0 * B[i][0]));
        const float n1 = fmaf(R2, B[i][7], fmaf(R1, B[i][4], R0 * B[i][1]));
        const float n2 = fmaf(R2, B[i][8], fmaf(R1, B[i][5], R0 * B[i][2]));
        R0 = n0; R1 = n1; R2 = n2;
        const int r = i * KC_BS + KB_R + 3 * u;
        s[r] = R0; s[r + 1] = R1; s[r + 2] = R2;
        s[i * KC_BS + KB_P + u] = p;
        if (i == 7) { S0 = R0; S1 = R1; S2 = R2; sp = p; }
    }
#undef KC_CHAIN_LOAD
}

// Phase 3: world-frame quantities of the lane's bodies + collision candidates of the lane's spheres.
template <bool TWOB, class S>
KC_F bool kc_ph_body(const S& s, const float* tab, const KukaParams& P, const KcKinIn& in, int u) {
#pragma unroll 1
    for (int k = 0; k < KK_NB / KC_G; ++k) {
        const int i = u + KC_G * k, o = i * KC_BS;
        const float* c = tab + i * KC_CS;
        float R[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) R[t] = s[o + KB_R + t];
        const kc3 p = kc_ld3(s, o + KB_P);
        const float ax = c[KCB_AXIS], ay = c[KCB_AXIS + 1], az = c[KCB_AXIS + 2];
        const float I0 = c[KCB_IC], I1 = c[KCB_IC + 1], I2 = c[KCB_IC + 2], I3 = c[KCB_IC + 3], I4 = c[KCB_IC + 4], I5 = c[KCB_IC + 5];
        const float m = c[KCB_MASS];    // (all loads ahead of the stores)
        const kc3 a = kc_mk(fmaf(R[2], az, fmaf(R[1], ay, R[0] * ax)), fmaf(R[5], az, fmaf(R[4], ay, R[3] * ax)), fmaf(R[8], az, fmaf(R[7], ay, R[6] * ax)));
        const float mx = c[KCB_COM], my = c[KCB_COM + 1], mz = c[KCB_COM + 2];
        const kc3 cm = kc_mk(fmaf(R[2], mz, fmaf(R[1], my, fmaf(R[0], mx, p.x))), fmaf(R[5], mz, fmaf(R[4], my, fmaf(R[3], mx, p.y))),
                             fmaf(R[8], mz, fmaf(R[7], my, fmaf(R[6], mx, p.z))));
        kc_st3(s, o + KB_A, a);
        kc_st3(s, o + KB_PV, kc_cross(p, a));
        kc_st3(s, o + KB_C, cm);
        // Iw = R Ic R^T
        float T[9];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            T[3 * r + 0] = fmaf(R[3 * r + 2], I2, fmaf(R[3 * r + 1], I1, R[3 * r] * I0));
            T[3 * r + 1] = fmaf(R[3 * r + 2], I4, fmaf(R[3 * r + 1], I3, R[3 * r] * I1));
            T[3 * r + 2] = fmaf(R[3 * r + 2], I5, fmaf(R[3 * r + 1], I4, R[3 * r] * I2));
        }
        float Iw[6];
        Iw[0] = fmaf(T[2], R[2], fmaf(T[1], R[1], T[0] * R[0]));
        Iw[1] = fmaf(T[2], R[5], fmaf(T[1], R[4], T[0] * R[3]));
        Iw[2] = fmaf(T[2], R[8], fmaf(T[1], R[7], T[0] * R[6]));
        Iw[3] = fmaf(T[5], R[5], fmaf(T[4], R[4], T[3] * R[3]));
        Iw[4] = fmaf(T[5], R[8], fmaf(T[4], R[7], T[3] * R[6]));
        Iw[5] = fmaf(T[8], R[8], fmaf(T[7], R[7], T[6] * R[6]));
#pragma unroll
        for (int t = 0; t < 6; ++t) s[o + KB_IW + t] = Iw[t];
        // spatial inertia about the world origin: m, h = m c, I_O = Iw + m (|c|^2 1 - c c^T)
        s[o + KB_M] = m;
        kc_st3(s, o + KB_H, kc_scale(m, cm));
        s[o + KB_IO + 0] = fmaf(m, fmaf(cm.y, cm.y, cm.z * cm.z), Iw[0]);
        s[o + KB_IO + 1] = fmaf(-m * cm.x, cm.y, Iw[1]);
        s[o + KB_IO + 2] = fmaf(-m * cm.x, cm.z, Iw[2]);
        s[o + KB_IO + 3] = fmaf(m, fmaf(cm.x, cm.x, cm.z * cm.z), Iw[3]);
        s[o + KB_IO + 4] = fmaf(-m * cm.y, cm.z, Iw[4]);
        s[o + KB_IO + 5] = fmaf(m, fmaf(cm.x, cm.x, cm.y * cm.y), Iw[5]);
    }
    // ---- collision detection: sphere vs {table, disc, stack [, disc 2, stack 2]}; skipped while the lowest sphere-carrying body frame is
    //      more than (reach + margin) above every shape -- most of an episode
    const float bz = in.bbz;
    const float disc0 = bz + P.glider_z + in.qb + P.disc_z0, disc1 = bz + P.glider_z + in.qb + P.disc_z1;
    const float b2z = P.btn_base[2];
    const float disc20 = b2z + P.glider_z + in.qb2 + P.disc_z0, disc21 = b2z + P.glider_z + in.qb2 + P.disc_z1;
    float zmax_shapes = fmaxf(disc1, fmaxf(bz + P.stack_top, P.table_z));
    if (TWOB) zmax_shapes = fmaxf(zmax_shapes, fmaxf(disc21, b2z + P.stack_top));
    float zmin_body = 1e30f;
#pragma unroll
    for (int i = 0; i < KK_NB; ++i)   // independent loads (a rolled loop waits for each)
        if (i >= P.sph_min_body) zmin_body = fminf(zmin_body, s[i * KC_BS + KB_P + 2]);
    const bool near = zmin_body - P.sph_reach - zmax_shapes <= P.cdist;
    if (!near) return false;    // (the same value in the 4 lanes) no candidate is written, the collect phase is skipped
#pragma unroll 1
    for (int sidx = u; sidx < P.nsph; sidx += KC_G) {
        const int cw = KC_OFF_CAND + sidx * KC_CANDW;
        int ncand = 0;
        {
            const float* sp = tab + KC_CONST_SPH + sidx * 5;
            const int b = (int)sp[0], o = b * KC_BS;
            const float r = sp[4];
            const float scz = fmaf(s[o + KB_R + 8], sp[3], fmaf(s[o + KB_R + 7], sp[2], fmaf(s[o + KB_R + 6], sp[1], s[o + KB_P + 2])));
            if (scz - r - zmax_shapes <= P.cdist) {   // cheap reject on z alone: well above every shape
                const kc3 sc = kc_mk(fmaf(s[o + KB_R + 2], sp[3], fmaf(s[o + KB_R + 1], sp[2], fmaf(s[o + KB_R + 0], sp[1], s[o + KB_P]))),
                                     fmaf(s[o + KB_R + 5], sp[3], fmaf(s[o + KB_R + 4], sp[2], fmaf(s[o + KB_R + 3], sp[1], s[o + KB_P + 1]))), scz);
#pragma unroll 1
                for (int shape = 0; shape < (TWOB ? 5 : 3); ++shape) {   // 0 table, 1 / 2 disc / stack of button 1, 3 / 4 of button 2
                    float dist; kc3 nn;
                    if (shape == 0) {
                        if (sc.x < P.txmin || sc.x > P.txmax || sc.y < P.tymin || sc.y > P.tymax) continue;
                        dist = sc.z - P.table_z - r; nn = kc_mk(0.f, 0.f, 1.f);
                    } else if (!TWOB || shape < 3) {
                        const float z0 = shape == 1 ? disc0 : bz, z1 = shape == 1 ? disc1 : bz + P.stack_top;
                        kc_sphere_cylinder(sc, r, in.bbx, in.bby, z0, z1, shape == 1 ? P.disc_r : P.stack_r, dist, nn);
                    } else {
                        const float z0 = shape == 3 ? disc20 : b2z, z1 = shape == 3 ? disc21 : b2z + P.stack_top;
                        kc_sphere_cylinder(sc, r, in.bb2x, in.bb2y, z0, z1, shape == 3 ? P.disc_r : P.stack_r, dist, nn);
                    }
                    if (dist > P.cdist) continue;
                    if (ncand < KC_CANDS) {
                        const int w = cw + 1 + ncand * 8;
                        s[w] = (float)shape; s[w + 1] = dist; kc_st3(s, w + 2, nn);
                        kc_st3(s, w + 5, kc_mk(fmaf(-r, nn.x, sc.x), fmaf(-r, nn.y, sc.y), fmaf(-r, nn.z, sc.z)));
                    }
                    ++ncand;      // a sphere cannot be within the margin of more than three of these shapes at once (the buttons are 25 cm apart)
                }
            }
        }
        s[cw] = (float)ncand;
    }
    return true;
}

// Phase 4 (lane 0; only when some sphere may be within the margin of a shape): manifold flags and the first max_contacts candidates in
// (sphere, shape) order -> contact records.
template <bool TWOB, class S>
KC_F void kc_ph_collect(const S& s, const float* tab, const KukaParams& P, int u) {
    if (u != 0) return;
    // the candidate counts of all spheres first (independent loads), then a walk over the few spheres that have any, in sphere order
    // (a walk that loads each count and branches on it waits for one shared-memory load per sphere)
    unsigned has = 0u;
#pragma unroll
    for (int sidx = 0; sidx < KM_MAX_SPHERES; ++sidx)
        if (sidx < P.nsph && s[KC_OFF_CAND + sidx * KC_CANDW] > 0.f) has |= 1u << sidx;
    int flags = 0, nc = 0;      // bit 0 button disc, 1 table, 2 any link of button 1, 3 any link of button 2
#pragma unroll 1
    for (; has != 0u; has &= has - 1u) {
        const int sidx = kc_lowest_bit(has);
        const int cw = KC_OFF_CAND + sidx * KC_CANDW;
        int ncand = (int)s[cw];
        if (ncand > KC_CANDS) ncand = KC_CANDS;
#pragma unroll 1
        for (int k = 0; k < ncand; ++k) {
            const int w = cw + 1 + k * 8;
            const int shape = (int)s[w];
            if (shape == 0) flags |= 2;
            if (shape == 1) flags |= 1;
            if (TWOB) { if (shape == 1 || shape == 2) flags |= 4; if (shape >= 3) flags |= 8; }
            if (nc < P.max_contacts && nc < KK_MAXC) {
                const int c = KC_OFF_CT + nc * KC_CTS;
                float rec[KC_CTS];      // loaded whole, then stored
                rec[0] = tab[KC_CONST_SPH + sidx * 5];
#pragma unroll
                for (int t = 0; t < 8; ++t) rec[1 + t] = s[w + t];
#pragma unroll
                for (int t = 0; t < KC_CTS; ++t) s[c + t] = rec[t];
                ++nc;
            }
        }
    }
    s[KC_OFF_LINK + 6] = (float)flags; s[KC_OFF_LINK + 7] = (float)nc;
}

// ================================================================ dynamics ========================================================
// Tree prefix sum of a 3-vector field: out_i = (root value) + sum over the ancestors-or-self j of term_j, one scalar component per call.
// Lanes 0..2 take components of the first field, lane 3 and lanes 0..1 (second pass) of the second: 6 scalars over 4 lanes.
template <class S>
KC_F void kc_prefix_scalar(const S& s, int field, int comp, float root) {
    float t[KK_NB];
#pragma unroll
    for (int i = 0; i < KK_NB; ++i) t[i] = s[i * KC_BS + field + comp];     // independent loads first, then the dependent adds
    float acc = root, acc7 = root;
#pragma unroll
    for (int i = 0; i < KK_NB; ++i) {
        if (i == 10) acc = acc7;
        acc += t[i];
        s[i * KC_BS + field + comp] = acc;
        if (i == 7) acc7 = acc;
    }
}

// Phase D1: terms qd_i a_i, qd_i pv_i of the lane's bodies (into W / VO).
template <class S>
KC_F void kc_ph_vel_terms(const S& s, const float* qd, int u) {
#pragma unroll
    for (int k = 0; k < KK_NB / KC_G; ++k) {
        const int o = (u + KC_G * k) * KC_BS;
        const float qdi = KC_SEL4(qd, k, u);
        kc_st3(s, o + KB_W, kc_scale(qdi, kc_ld3(s, o + KB_A)));
        kc_st3(s, o + KB_VO, kc_scale(qdi, kc_ld3(s, o + KB_PV)));
    }
}
// Phase D2 / D4: prefix sums of two 3-vector fields (6 scalars: lanes 0, 1 take two, lanes 2, 3 one).
template <class S>
KC_F void kc_ph_prefix2(const S& s, int f0, int f1, float root1z, int u) {
    kc_prefix_scalar(s, u < 3 ? f0 : f1, u < 3 ? u : 0, 0.f);
    if (u < 2) kc_prefix_scalar(s, f1, 1 + u, u == 1 ? root1z : 0.f);
}
// Phase D3: acceleration terms of the lane's bodies: qd_i (w_p x a_i), qd_i (w_p x pv_i + vO_p x a_i) with the PARENT's velocities.
template <class S>
KC_F void kc_ph_acc_terms(const S& s, const float* qd, int u) {
#pragma unroll
    for (int k = 0; k < KK_NB / KC_G; ++k) {
        const int i = u + KC_G * k, o = i * KC_BS, pa = kc_parent(i);
        const float qdi = KC_SEL4(qd, k, u);
        kc3 wp = kc_mk(0.f, 0.f, 0.f), vp = wp;
        if (pa >= 0) { wp = kc_ld3(s, pa * KC_BS + KB_W); vp = kc_ld3(s, pa * KC_BS + KB_VO); }
        const kc3 a = kc_ld3(s, o + KB_A), pv = kc_ld3(s, o + KB_PV);
        kc_st3(s, o + KB_AW, kc_scale(qdi, kc_cross(wp, a)));
        kc_st3(s, o + KB_AV, kc_scale(qdi, kc_add(kc_cross(wp, pv), kc_cross(vp, a))));
    }
}
// Phase D5: wrench of the lane's bodies about the world origin (inertial + velocity-product + Bullet link damping).
template <class S>
KC_F void kc_ph_wrench(const S& s, const KukaParams& P, int u) {
#pragma unroll 1
    for (int k = 0; k < KK_NB / KC_G; ++k) {
        const int o = (u + KC_G * k) * KC_BS;
        const kc3 w = kc_ld3(s, o + KB_W), vO = kc_ld3(s, o + KB_VO), aw = kc_ld3(s, o + KB_AW), av = kc_ld3(s, o + KB_AV);
        const kc3 c = kc_ld3(s, o + KB_C), h = kc_ld3(s, o + KB_H);
        const float m = s[o + KB_M];
        float IO[6], Iw[6];
#pragma unroll
        for (int t = 0; t < 6; ++t) { IO[t] = s[o + KB_IO + t]; Iw[t] = s[o + KB_IW + t]; }
        const kc3 Lv = kc_add(kc_symv(IO, w), kc_cross(h, vO));
        const kc3 Pv = kc_fma(m, vO, kc_cross(w, h));
        const kc3 La = kc_add(kc_symv(IO, aw), kc_cross(h, av));
        const kc3 Pa = kc_fma(m, av, kc_cross(aw, h));
        kc3 n = kc_add(kc_add(La, kc_cross(w, Lv)), kc_cross(vO, Pv));
        kc3 f = kc_add(Pa, kc_cross(w, Pv));
        // btMultiBody link damping (linear / angular 0.04, K1 = K2): resisting wrench added to the bias
        const kc3 vc = kc_add(vO, kc_cross(w, c));
        const kc3 F = kc_scale(P.kl * m * (1.0f + sqrtf(kc_dot(vc, vc))), vc);
        const kc3 T = kc_scale(P.ka * (1.0f + sqrtf(kc_dot(w, w))), kc_symv(Iw, w));
        n = kc_add(kc_add(n, T), kc_cross(c, F));
        f = kc_add(f, F);
        kc_st3(s, o + KB_N, n);
        kc_st3(s, o + KB_F, f);
    }
}
// Phase D6: sub-tree sums of the 16 scalars (m, h, IO, n, f) -- 4 scalars per lane, leaves first (the order the serial code adds them in).
template <class S>
KC_F void kc_ph_subtree(const S& s, int u) {
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const int idx = 4 * u + t;                            // 0..15
        const int f = idx < 10 ? KB_M + idx : KB_N + (idx - 10);   // M, H[3], IO[6] are contiguous from KB_M; N[3], F[3] from KB_N
        float v[KK_NB];
#pragma unroll
        for (int j = 0; j < KK_NB; ++j) v[j] = s[j * KC_BS + f];
#pragma unroll
        for (int j = KK_NB - 1; j >= 1; --j) v[j == 10 ? 7 : j - 1] += v[j];        // parent += child, children in descending order
#pragma unroll
        for (int j = 0; j < KK_NB - 1; ++j)
            if (j != 9) s[j * KC_BS + f] = v[j];                                    // bodies 9 and 11 are leaves
    }
}
// Phase D7: bias torque, momentum vectors and ROW j of the mass matrix for the lane's bodies j (lower triangle; non-ancestor entries are
// zero).  Axes and motion vectors of all 12 bodies are read once (compile-time addresses, independent loads); the row is 12 predicated
// dot products on registers.
template <class S>
KC_F void kc_ph_mass(const S& s, int u) {
    kc3 a[KK_NB], pv[KK_NB];
#pragma unroll
    for (int i = 0; i < KK_NB; ++i) { a[i] = kc_ld3(s, i * KC_BS + KB_A); pv[i] = kc_ld3(s, i * KC_BS + KB_PV); }
#pragma unroll
    for (int k = 0; k < KK_NB / KC_G; ++k) {
        const int j = u + KC_G * k, o = j * KC_BS;
        const kc3 aj = kc_ld3(s, o + KB_A), pvj = kc_ld3(s, o + KB_PV);   // (a[j] with a run-time j would put the arrays in local memory)
        const kc3 h = kc_ld3(s, o + KB_H);
        s[KC_OFF_BIAS + j] = kc_dot(aj, kc_ld3(s, o + KB_N)) + kc_dot(pvj, kc_ld3(s, o + KB_F));
        float I[6];
#pragma unroll
        for (int t = 0; t < 6; ++t) I[t] = s[o + KB_IO + t];
        const kc3 Pm = kc_fma(s[o + KB_M], pvj, kc_cross(aj, h));      // linear momentum of the composite under unit joint rate
        const kc3 Lm = kc_add(kc_symv(I, aj), kc_cross(h, pvj));        // angular momentum about the origin
#pragma unroll
        for (int i = 0; i < KK_NB; ++i) {
            if (i > 4 * k + 3) continue;                               // above the diagonal for every j = 4 k + u
            const float val = kc_anc(i, j) ? kc_dot(a[i], Lm) + kc_dot(pv[i], Pm) : 0.f;
            if (i < 4 * k || i <= j) s[KC_OFF_MA + j * KC_MS + i] = val;   // i <= j (only u is a run-time value)
        }
    }
}

// Phase C1 (A = M^-1 in registers, lower triangle valid, UNSCALED): constraint rows of the contact manifold -- Jacobian, W = M^-1 J^T, 1 / D,
// target -- row r -> lane r & 3, in the KK_ROW_* layout.  SCALED: stored for the scaled system of the sweeps (kuka_physics_step): J_j / sigma_j
// and sigma_j W_j on the 12 arm DoF, target - J . tgt (tgt = the motor rows' target velocities).
template <bool TWOB, bool SCALED, class S>
KC_F void kc_ph_rows(const S& s, const KukaParams& P, const float (&A)[KK_NB][KK_NB], int nc, int u, const float* tgt = nullptr) {
#pragma unroll 1
    for (int r = u; r < 3 * nc; r += KC_G) {
        const int c = r < nc ? r : (r - nc) >> 1;
        const int co = KC_OFF_CT + c * KC_CTS, ro = KC_OFF_ROWS + r * KC_RS;
        const kc3 n = kc_ld3(s, co + 3), pt = kc_ld3(s, co + 6);
        kc3 dir = n;
        if (r >= nc) {  // btPlaneSpace1 tangents
            kc3 t1, t2;
            if (fabsf(n.z) > 0.70710678f) {
                const float a = n.y * n.y + n.z * n.z, kk = KC_RSQRT(a);
                t1 = kc_mk(0.f, -n.z * kk, n.y * kk); t2 = kc_mk(a * kk, -n.x * t1.z, n.x * t1.y);
            } else {
                const float a = n.x * n.x + n.y * n.y, kk = KC_RSQRT(a);
                t1 = kc_mk(-n.y * kk, n.x * kk, 0.f); t2 = kc_mk(-n.z * t1.y, n.z * t1.x, a * kk);
            }
            dir = ((r - nc) & 1) ? t2 : t1;
        }
        const int body = (int)s[co], shape = (int)s[co + 1];
        float J[KK_NB];
#pragma unroll
        for (int j = 0; j < KK_NB; ++j)
            J[j] = kc_anc(j, body) ? kc_dot(dir, kc_cross(kc_ld3(s, j * KC_BS + KB_A), kc_sub(pt, kc_ld3(s, j * KC_BS + KB_P)))) : 0.f;
        const float jb = shape == 1 ? -dir.z : 0.f, jb2 = TWOB && shape == 3 ? -dir.z : 0.f;
        float D = 0.f, off = 0.f;
#pragma unroll
        for (int i = 0; i < KK_NB; ++i) {
            float acc = 0.f;
#pragma unroll
            for (int j = 0; j < KK_NB; ++j) acc = fmaf(i >= j ? A[i][j] : A[j][i], J[j], acc);
            D = fmaf(J[i], acc, D);
            if (SCALED) off = fmaf(J[i], tgt[i], off);
            s[ro + KK_ROW_J + i] = SCALED ? J[i] * P.sat_isig[i] : J[i];
            s[ro + KK_ROW_W + i] = SCALED ? acc * P.sat_sig[i] : acc;
            if (SCALED && r < nc) s[KC_OFF_WT + 4 * i + r] = acc * P.sat_sig[i];     // the watch matrix column of this normal row
        }
        s[ro + KK_ROW_J + KK_NB] = jb; s[ro + KK_ROW_W + KK_NB] = jb * P.btn_minv;
        s[ro + KK_ROW_J + KK_NB + 1] = jb2; s[ro + KK_ROW_W + KK_NB + 1] = jb2 * P.btn_minv;
        D = fmaf(jb, jb * P.btn_minv, D);
        if (TWOB) D = fmaf(jb2, jb2 * P.btn_minv, D);
        s[ro + KK_ROW_INVD] = 1.0f / D;
        const float pen = s[co + 2];
        s[ro + KK_ROW_TGT] = (r < nc ? (pen > 0.f ? -pen * P.inv_dt : -P.erp * pen * P.inv_dt) : 0.f) - off;
    }
}

// ================================================================ drivers =========================================================
// On the device every lane of the group calls the phase with its own u and the group meets at __syncwarp(); on the host the caller's
// KC_RUN runs the 4 lanes one after the other.
#if defined(__CUDACC__)
#define KC_RUN(call) do { call; __syncwarp(gmask); } while (0)      // gmask: the 4 lanes of the group
#else
#define KC_RUN(call) do { for (int u = 0; u < KC_G; ++u) { call; } } while (0)
#endif

// Returns whether the contact manifold had to be looked at (false: no flag set, no contact record); the link states are fields of the
// body records (COM of link 8, origin of link 6).
#if defined(__CUDACC__)
template <bool TWOB, class S>
KC_F bool kc_kinematics(const S& s, const float* tab, const KukaParams& P, const KcKinIn& in, int u, unsigned gmask, KkPhaseClock* ph) {
    KC_RUN(kc_ph_local(s, tab, in, u));
    KK_PH(ph, KK_PH_KIN_LOCAL);
    KC_RUN(kc_ph_chain(s, tab, P, u));
    KK_PH(ph, KK_PH_KIN_CHAIN);
    const bool near = kc_ph_body<TWOB>(s, tab, P, in, u);
    __syncwarp(gmask);
    KK_PH(ph, KK_PH_KIN_BODY);
    if (near) KC_RUN((kc_ph_collect<TWOB>(s, tab, P, u)));
    return near;
}
#else
template <bool TWOB, class S>
KC_F bool kc_kinematics(const S& s, const float* tab, const KukaParams& P, const KcKinIn& in) {
    KC_RUN(kc_ph_local(s, tab, in, u));
    KC_RUN(kc_ph_chain(s, tab, P, u));
    bool near = false;
    for (int u = 0; u < KC_G; ++u) near = kc_ph_body<TWOB>(s, tab, P, in, u);
    if (near) KC_RUN((kc_ph_collect<TWOB>(s, tab, P, u)));
    return near;
}
#endif

#if defined(__CUDACC__)
template <class S>
KC_F void kc_dynamics(const S& s, const KukaParams& P, const float* qd, int u, unsigned gmask, KkPhaseClock* ph) {
#else
template <class S>
KC_F void kc_dynamics(const S& s, const KukaParams& P, const float* qd) {
    KkPhaseClock* const ph = nullptr;
#endif
    KC_RUN(kc_ph_vel_terms(s, qd, u));
    KK_PH(ph, KK_PH_DYN_D1);
    KC_RUN(kc_ph_prefix2(s, KB_W, KB_VO, 0.f, u));
    KK_PH(ph, KK_PH_DYN_D2);
    KC_RUN(kc_ph_acc_terms(s, qd, u));
    KK_PH(ph, KK_PH_DYN_D3);
    KC_RUN(kc_ph_prefix2(s, KB_AW, KB_AV, -P.gz, u));      // gravity as a fictitious base acceleration
    KK_PH(ph, KK_PH_DYN_D4);
    KC_RUN(kc_ph_wrench(s, P, u));
    KK_PH(ph, KK_PH_DYN_D5);
    KC_RUN(kc_ph_subtree(s, u));
    KK_PH(ph, KK_PH_DYN_D6);
    KC_RUN(kc_ph_mass(s, u));
}
