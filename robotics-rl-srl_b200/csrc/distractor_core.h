// KukaRandButtonGymEnv's distractor bodies (kuka_rand_button_gym_env.py:58-68,117-127): up to 10 objects dropped on the table
// plus the small sphere that is kicked at env step 10.  One header for both sides: the CUDA library instantiates it in float
// (distractor_kernel, distractor_kernels.cu) and the float64 CPU checker (distractor_ref.cpp) in double.
//
// Model (DESIGN.md section 4, "Distractor bodies"):
//   * free 6-DoF bodies, gravity -g along z, time step dt; no damping, no sleeping, no rolling friction;
//   * collision geometry = a compound of at most DC_MAXSPH spheres per body (the pybullet_data meshes are not available);
//   * contacts against the table top (a box top: the sphere must lie over the table's x / y extent), the button's base stack and
//     disc (upright cylinders; the disc follows the glider), the arm's collision spheres, and the spheres of the other bodies;
//     a contact exists when the distance is <= margin (0.02 m, Bullet's manifold margin);
//   * rows: one normal (target -dist/dt when separated, -0.2 dist/dt when penetrating, lambda >= 0) and two friction rows
//     (|lambda| <= mu lambda_n, mu = product of the two surfaces' coefficients) per contact, projected Gauss-Seidel over all rows
//     for `iters` sweeps without warm start, then semi-implicit Euler with quaternion integration;
//   * ONE-WAY coupling: the arm, the button and the table are kinematic for the bodies -- the arm's solve never sees them.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define DC_HD __host__ __device__ __forceinline__
#else
#define DC_HD inline
#endif

#define DC_NBODY 11        // 10 placement slots + the kicked sphere (slot 10)
#define DC_NTYPE 4         // 0 duck_vhacd, 1 lego, 2 cube_small, 3 sphere_small
#define DC_MAXSPH 4        // collision spheres per body
#define DC_MAXC 48         // contacts per island and micro-step (further contacts are dropped)
#define DC_MAXARM 16       // arm collision spheres

// asset blob: f64[DC_NTYPE][DC_TYPE_WORDS] (srl_sim/model.py: distractor_blob)
#define DC_TYPE_WORDS 32
enum {
    DC_A_MASS = 0, DC_A_INERTIA = 1 /* Ixx Iyy Izz about the COM = link origin */, DC_A_MU = 4, DC_A_NSPH = 5,
    DC_A_SPH = 6 /* DC_MAXSPH x (cx, cy, cz, r) */, DC_A_HALF = 22 /* rendering: half extents */, DC_A_RGB = 25, DC_A_SHAPE = 28 /* 0 box 1 sphere */
};
#define DC_BLOB_WORDS (DC_NTYPE * DC_TYPE_WORDS)

// per body, f32[16] in HBM / f64[16] on the CPU side
enum { DC_B_P = 0, DC_B_Q = 3 /* x y z w */, DC_B_V = 7, DC_B_W = 10, DC_B_TYPE = 13, DC_B_PRESENT = 14, DC_B_WORDS = 16 };

// placement constants of the reference (kuka_rand_button_gym_env.py:58-66), Z_TABLE = -0.2 (kuka_button_gym_env.py:26)
#define DC_Z_TABLE (-0.2)
#define DC_DROP_H 0.1
#define DC_SPHERE_X 0.25
#define DC_SPHERE_Y (-0.2)
#define DC_SPHERE_H 0.3
#define DC_BALL_FORCE 10.0
#define DC_STATIC_MU 1.0   // table, button and arm surfaces (RECALLED: pybullet's default lateral friction)

template <class R> struct DcType { R m, inv_m, inv_I[3], mu; int nsph; R c[DC_MAXSPH][3]; R r[DC_MAXSPH]; };
template <class R> struct DcAssets { DcType<R> t[DC_NTYPE]; };

// scene of one micro-step: static geometry + the kinematic button and arm
template <class R> struct DcScene {
    R table_z, txmin, txmax, tymin, tymax;
    R bx, by, bz, stack_top, stack_r, disc_r, disc0, disc1;   // disc0 / disc1: absolute z range of the disc this micro-step
    R dt, g, margin;
    int iters;
};

template <class R> DC_HD void dc_assets_from_blob(const double* b, DcAssets<R>& A) {
    for (int t = 0; t < DC_NTYPE; ++t) {
        const double* w = b + t * DC_TYPE_WORDS;
        DcType<R>& T = A.t[t];
        T.m = (R)w[DC_A_MASS]; T.inv_m = (R)(1.0 / w[DC_A_MASS]);
        for (int a = 0; a < 3; ++a) T.inv_I[a] = (R)(1.0 / w[DC_A_INERTIA + a]);
        T.mu = (R)w[DC_A_MU];
        T.nsph = (int)w[DC_A_NSPH];
        for (int s = 0; s < DC_MAXSPH; ++s) {
            for (int a = 0; a < 3; ++a) T.c[s][a] = (R)w[DC_A_SPH + 4 * s + a];
            T.r[s] = (R)w[DC_A_SPH + 4 * s + 3];
        }
    }
}

// checks a blob; returns an error message or nullptr
DC_HD const char* dc_blob_error(const double* b, size_t bytes) {
    if (bytes != DC_BLOB_WORDS * sizeof(double)) return "distractor asset blob: wrong size";
    for (int t = 0; t < DC_NTYPE; ++t) {
        const double* w = b + t * DC_TYPE_WORDS;
        if (!(w[DC_A_MASS] > 0.0) || !(w[DC_A_INERTIA] > 0.0) || !(w[DC_A_INERTIA + 1] > 0.0) || !(w[DC_A_INERTIA + 2] > 0.0))
            return "distractor asset blob: mass and inertia must be positive";
        if (!(w[DC_A_NSPH] >= 1.0 && w[DC_A_NSPH] <= DC_MAXSPH)) return "distractor asset blob: 1 to 4 collision spheres per body";
        if (!(w[DC_A_MU] >= 0.0)) return "distractor asset blob: negative friction";
        // the drawing words (render_core.h: srl_distractor_prims)
        if (!(w[DC_A_SHAPE] == 0.0 || w[DC_A_SHAPE] == 1.0)) return "distractor asset blob: DC_A_SHAPE must be 0 (box) or 1 (sphere)";
        for (int a = 0; a < 3; ++a) {
            if (!(w[DC_A_HALF + a] > 0.0)) return "distractor asset blob: DC_A_HALF (half extents) must be positive";
            if (!(w[DC_A_RGB + a] >= 0.0 && w[DC_A_RGB + a] <= 1.0)) return "distractor asset blob: DC_A_RGB must lie in [0, 1]";
        }
    }
    return nullptr;
}

// rotation matrix of a unit quaternion (x, y, z, w)
template <class R> DC_HD void dc_rot(const R* q, R* M) {
    const R x = q[0], y = q[1], z = q[2], w = q[3];
    M[0] = 1 - 2 * (y * y + z * z); M[1] = 2 * (x * y - z * w);     M[2] = 2 * (x * z + y * w);
    M[3] = 2 * (x * y + z * w);     M[4] = 1 - 2 * (x * x + z * z); M[5] = 2 * (y * z - x * w);
    M[6] = 2 * (x * z - y * w);     M[7] = 2 * (y * z + x * w);     M[8] = 1 - 2 * (x * x + y * y);
}

// reset(): body k of the 10 placement slots at (x_k, y_k) unless inside the +-0.1 square around the button (:62-66), the sphere
// always; `type[k]` in 0..2 (rand_objects[np.random.randint(3)]).  Bodies start at rest, unrotated.
template <class R> DC_HD void dc_place(R* B, const double* xy /*[20]*/, const int* type /*[10]*/, double btn_x, double btn_y) {
    for (int k = 0; k < DC_NBODY; ++k) {
        R* b = B + k * DC_B_WORDS;
        for (int j = 0; j < DC_B_WORDS; ++j) b[j] = (R)0;
        b[DC_B_Q + 3] = (R)1;
        if (k < 10) {
            const double x = xy[2 * k], y = xy[2 * k + 1];
            const bool out = (x < btn_x - 0.1) || (x > btn_x + 0.1) || (y < btn_y - 0.1) || (y > btn_y + 0.1);
            b[DC_B_P] = (R)x; b[DC_B_P + 1] = (R)y; b[DC_B_P + 2] = (R)(DC_Z_TABLE + DC_DROP_H);
            b[DC_B_TYPE] = (R)type[k]; b[DC_B_PRESENT] = out ? (R)1 : (R)0;
        } else {
            b[DC_B_P] = (R)DC_SPHERE_X; b[DC_B_P + 1] = (R)DC_SPHERE_Y; b[DC_B_P + 2] = (R)(DC_Z_TABLE + DC_SPHERE_H);
            b[DC_B_TYPE] = (R)3; b[DC_B_PRESENT] = (R)1;
        }
    }
}

// sphere (centre s, radius r) vs upright cylinder: signed distance and normal from the cylinder towards the sphere
template <class R> DC_HD void dc_sphere_cyl(const R* s, R r, R cx, R cy, R z0, R z1, R rad, R& dist, R* n) {
    const R dx = s[0] - cx, dy = s[1] - cy;
    const R rho = sqrt(dx * dx + dy * dy);
    const R ux = rho > (R)1e-12 ? dx / rho : (R)1, uy = rho > (R)1e-12 ? dy / rho : (R)0;
    R d;
    n[0] = 0; n[1] = 0; n[2] = 0;
    if (s[2] >= z1 || s[2] <= z0) {
        const R zc = s[2] >= z1 ? z1 : z0;
        if (rho <= rad) { d = s[2] >= z1 ? s[2] - z1 : z0 - s[2]; n[2] = s[2] >= z1 ? (R)1 : (R)-1; }
        else {
            const R vx = dx - ux * rad, vy = dy - uy * rad, vz = s[2] - zc;
            d = sqrt(vx * vx + vy * vy + vz * vz);
            n[0] = vx / d; n[1] = vy / d; n[2] = vz / d;
        }
    } else if (rho > rad) { d = rho - rad; n[0] = ux; n[1] = uy; }
    else {
        const R dtop = z1 - s[2], dside = rad - rho;
        if (dtop <= dside) { d = -dtop; n[2] = 1; } else { d = -dside; n[0] = ux; n[1] = uy; }
    }
    dist = d - r;
}

// btPlaneSpace1
template <class R> DC_HD void dc_plane_space(const R* n, R* p, R* q) {
    if (fabs(n[2]) > (R)0.7071067811865475) {
        const R a = n[1] * n[1] + n[2] * n[2], k = (R)1 / sqrt(a);
        p[0] = 0; p[1] = -n[2] * k; p[2] = n[1] * k;
        q[0] = a * k; q[1] = -n[0] * p[2]; q[2] = n[0] * p[1];
    } else {
        const R a = n[0] * n[0] + n[1] * n[1], k = (R)1 / sqrt(a);
        p[0] = -n[1] * k; p[1] = n[0] * k; p[2] = 0;
        q[0] = -n[2] * p[1]; q[1] = n[2] * p[0]; q[2] = a * k;
    }
}

template <class R> struct DcRow {
    R d[3], ca[3], cb[3], ka[3], kb[3];   // direction, r_a x d, r_b x d, I_a^-1 (r_a x d), I_b^-1 (r_b x d)
    R inv_d, target, lambda, mu;
    int a, b, parent;                     // b < 0: kinematic partner; parent >= 0: friction row of normal row `parent`
};

template <class R> DC_HD R dc_dot(const R* a, const R* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
template <class R> DC_HD void dc_cross(const R* a, const R* b, R* c) {
    c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}

struct DcTouch { uint32_t body, arm; };   // per body bit masks of what it touched since the last placement: other bodies / the arm

// world collision spheres and world inverse inertia of every body of one env (shared by the phases of a micro-step)
template <class R> struct DcWork { R wc[DC_NBODY][DC_MAXSPH][3]; R Iw[DC_NBODY][9]; };

// A micro-step in phases, so that one lane per body can run it (distractor_kernel) and the CPU checker runs the same arithmetic in
// one thread (dc_step):
//   1. dc_prepare(k)       per body: world spheres, world inverse inertia, unconstrained velocity (gravity, the kick)
//   2. dc_adjacency(k)     per body: which bodies m > k are within the contact margin of body k
//   3. dc_island_roots     the bodies linked by body-body contacts form islands; the root of an island is its lowest slot
//   4. dc_island_solve(r)  per island: contact rows of its bodies in slot order, then the projected Gauss-Seidel sweeps
//   5. dc_integrate(k)     per body: semi-implicit Euler
// Gauss-Seidel over all rows of an env is island-by-island Gauss-Seidel: rows of different islands act on different bodies, so their
// order between islands does not matter and each island can be solved by its own lane with the same results.
// Contacts are capped at DC_MAXC per island (further contacts are dropped).

template <class R> DC_HD void dc_prepare(const DcAssets<R>& A, R* B, int k, DcWork<R>& W, const R* kick, const DcScene<R>& S) {
    R* b = B + k * DC_B_WORDS;
    if (b[DC_B_PRESENT] == (R)0) return;
    const DcType<R>& T = A.t[(int)b[DC_B_TYPE]];
    R M[9]; dc_rot(b + DC_B_Q, M);
    for (int s = 0; s < T.nsph; ++s)
        for (int r = 0; r < 3; ++r) W.wc[k][s][r] = b[DC_B_P + r] + M[3 * r] * T.c[s][0] + M[3 * r + 1] * T.c[s][1] + M[3 * r + 2] * T.c[s][2];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) W.Iw[k][3 * r + c] = M[3 * r] * T.inv_I[0] * M[3 * c] + M[3 * r + 1] * T.inv_I[1] * M[3 * c + 1] + M[3 * r + 2] * T.inv_I[2] * M[3 * c + 2];
    b[DC_B_V + 2] -= S.g * S.dt;
    if (kick && k == 10) {
        // applyExternalForce(sphere, -1, force, [0, 0, 0], WORLD_FRAME) (:125) acts at the WORLD ORIGIN: the impulse J gives the
        // ball J / m and the angular impulse (0 - p) x J
        for (int r = 0; r < 3; ++r) b[DC_B_V + r] += kick[r] * T.inv_m;
        const R arm_[3] = {-b[DC_B_P], -b[DC_B_P + 1], -b[DC_B_P + 2]};
        R L[3]; dc_cross(arm_, kick, L);
        for (int r = 0; r < 3; ++r) b[DC_B_W + r] += W.Iw[k][3 * r] * L[0] + W.Iw[k][3 * r + 1] * L[1] + W.Iw[k][3 * r + 2] * L[2];
    }
}

template <class R> DC_HD uint32_t dc_adjacency(const DcAssets<R>& A, const DcScene<R>& S, const R* B, const DcWork<R>& W, int k) {
    uint32_t adj = 0u;
    if (B[k * DC_B_WORDS + DC_B_PRESENT] == (R)0) return adj;
    const DcType<R>& T = A.t[(int)B[k * DC_B_WORDS + DC_B_TYPE]];
    for (int m = k + 1; m < DC_NBODY; ++m) {
        const R* bm = B + m * DC_B_WORDS;
        if (bm[DC_B_PRESENT] == (R)0) continue;
        const DcType<R>& Tm = A.t[(int)bm[DC_B_TYPE]];
        for (int s = 0; s < T.nsph; ++s)
            for (int s2 = 0; s2 < Tm.nsph; ++s2) {
                const R v[3] = {W.wc[k][s][0] - W.wc[m][s2][0], W.wc[k][s][1] - W.wc[m][s2][1], W.wc[k][s][2] - W.wc[m][s2][2]};
                if (sqrt(dc_dot(v, v)) - T.r[s] - Tm.r[s2] <= S.margin) adj |= 1u << m;
            }
    }
    return adj;
}

// root[k] = lowest slot of the island of body k
DC_HD void dc_island_roots(const uint32_t* adj, int* root) {
    for (int k = 0; k < DC_NBODY; ++k) root[k] = k;
    for (int pass = 0; pass < DC_NBODY; ++pass) {
        bool changed = false;
        for (int k = 0; k < DC_NBODY; ++k)
            for (int m = k + 1; m < DC_NBODY; ++m)
                if ((adj[k] >> m) & 1u) {
                    const int r = root[k] < root[m] ? root[k] : root[m];
                    if (root[k] != r || root[m] != r) { root[k] = r; root[m] = r; changed = true; }
                }
        if (!changed) break;
    }
}

// rows of the island rooted at `r` (bodies in slot order), then `iters` projected Gauss-Seidel sweeps over them
template <class R>
DC_HD void dc_island_solve(const DcAssets<R>& A, const DcScene<R>& S, R* B, const DcWork<R>& W, int r, const int* root, const R* arm, int narm,
                           DcRow<R>* rows, DcTouch* touch) {
    int nr = 0;
    auto add = [&](int a, int sa, int bb, const R* pb_world /*contact point on b, or null*/, const R* n, R dist) {
        if (nr + 3 > 3 * DC_MAXC) return;
        const R* pa = B + a * DC_B_WORDS;
        const DcType<R>& Ta = A.t[(int)pa[DC_B_TYPE]];
        // contact point on the surface of sphere sa of body a
        R ra[3], rb[3] = {0, 0, 0};
        for (int q = 0; q < 3; ++q) ra[q] = W.wc[a][sa][q] - Ta.r[sa] * n[q] - pa[DC_B_P + q];
        R mu = Ta.mu;
        if (bb >= 0) {
            const R* pbb = B + bb * DC_B_WORDS;
            for (int q = 0; q < 3; ++q) rb[q] = pb_world[q] - pbb[DC_B_P + q];
            mu *= A.t[(int)pbb[DC_B_TYPE]].mu;
        } else mu *= (R)DC_STATIC_MU;
        R t1[3], t2[3]; dc_plane_space(n, t1, t2);
        const R* dirs[3] = {n, t1, t2};
        const int first = nr;
        for (int j = 0; j < 3; ++j) {
            DcRow<R>& w = rows[nr++];
            for (int q = 0; q < 3; ++q) w.d[q] = dirs[j][q];
            dc_cross(ra, w.d, w.ca); dc_cross(rb, w.d, w.cb);
            for (int q = 0; q < 3; ++q) {
                w.ka[q] = W.Iw[a][3 * q] * w.ca[0] + W.Iw[a][3 * q + 1] * w.ca[1] + W.Iw[a][3 * q + 2] * w.ca[2];
                w.kb[q] = bb >= 0 ? W.Iw[bb][3 * q] * w.cb[0] + W.Iw[bb][3 * q + 1] * w.cb[1] + W.Iw[bb][3 * q + 2] * w.cb[2] : (R)0;
            }
            R den = Ta.inv_m + dc_dot(w.ca, w.ka);
            if (bb >= 0) den += A.t[(int)B[bb * DC_B_WORDS + DC_B_TYPE]].inv_m + dc_dot(w.cb, w.kb);
            w.inv_d = (R)1 / den;
            w.target = j ? (R)0 : (dist > 0 ? -dist / S.dt : (R)-0.2 * dist / S.dt);
            w.lambda = 0; w.mu = mu; w.a = a; w.b = bb; w.parent = j ? first : -1;
        }
    };
    // narrow phase
    for (int k = r; k < DC_NBODY; ++k) {
        if (root[k] != r) continue;
        const R* b = B + k * DC_B_WORDS;
        if (b[DC_B_PRESENT] == (R)0) continue;
        const DcType<R>& T = A.t[(int)b[DC_B_TYPE]];
        for (int s = 0; s < T.nsph; ++s) {
            const R* c = W.wc[k][s]; const R rad = T.r[s];
            R n[3], dist;
            // table top
            if (c[0] >= S.txmin && c[0] <= S.txmax && c[1] >= S.tymin && c[1] <= S.tymax) {
                dist = c[2] - S.table_z - rad;
                if (dist <= S.margin) { n[0] = 0; n[1] = 0; n[2] = 1; add(k, s, -1, nullptr, n, dist); }
            }
            // button disc and base stack
            dc_sphere_cyl(c, rad, S.bx, S.by, S.disc0, S.disc1, S.disc_r, dist, n);
            if (dist <= S.margin) add(k, s, -1, nullptr, n, dist);
            dc_sphere_cyl(c, rad, S.bx, S.by, S.bz, S.bz + S.stack_top, S.stack_r, dist, n);
            if (dist <= S.margin) add(k, s, -1, nullptr, n, dist);
            // arm spheres
            for (int j = 0; j < narm; ++j) {
                const R* ac = arm + 4 * j;
                const R v[3] = {c[0] - ac[0], c[1] - ac[1], c[2] - ac[2]};
                const R l = sqrt(dc_dot(v, v));
                dist = l - rad - ac[3];
                if (dist <= S.margin && l > (R)1e-9) {
                    n[0] = v[0] / l; n[1] = v[1] / l; n[2] = v[2] / l;
                    add(k, s, -1, nullptr, n, dist);
                    if (touch) touch->arm |= 1u << k;
                }
            }
            // the other bodies (each pair once: k < m; a body in contact is in the same island)
            for (int m = k + 1; m < DC_NBODY; ++m) {
                const R* bm = B + m * DC_B_WORDS;
                if (bm[DC_B_PRESENT] == (R)0 || root[m] != r) continue;
                const DcType<R>& Tm = A.t[(int)bm[DC_B_TYPE]];
                for (int s2 = 0; s2 < Tm.nsph; ++s2) {
                    const R* c2 = W.wc[m][s2];
                    const R v[3] = {c[0] - c2[0], c[1] - c2[1], c[2] - c2[2]};
                    const R l = sqrt(dc_dot(v, v));
                    dist = l - rad - Tm.r[s2];
                    if (dist <= S.margin && l > (R)1e-9) {
                        n[0] = v[0] / l; n[1] = v[1] / l; n[2] = v[2] / l;
                        const R pb[3] = {c2[0] + Tm.r[s2] * n[0], c2[1] + Tm.r[s2] * n[1], c2[2] + Tm.r[s2] * n[2]};
                        add(k, s, m, pb, n, dist);
                        if (touch) touch->body |= (1u << k) | (1u << m);
                    }
                }
            }
        }
    }
    // projected Gauss-Seidel on the velocities
    for (int it = 0; it < S.iters; ++it) {
        for (int j = 0; j < nr; ++j) {
            DcRow<R>& w = rows[j];
            R* va = B + w.a * DC_B_WORDS + DC_B_V;
            R vrel = dc_dot(w.d, va) + dc_dot(w.ca, va + 3);
            R* vb = nullptr;
            if (w.b >= 0) { vb = B + w.b * DC_B_WORDS + DC_B_V; vrel -= dc_dot(w.d, vb) + dc_dot(w.cb, vb + 3); }
            R lo = 0, hi = (R)1e30;
            if (w.parent >= 0) { hi = w.mu * rows[w.parent].lambda; lo = -hi; }
            R lnew = w.lambda + w.inv_d * (w.target - vrel);
            lnew = lnew < lo ? lo : (lnew > hi ? hi : lnew);
            const R dl = lnew - w.lambda;
            w.lambda = lnew;
            const R ima = A.t[(int)B[w.a * DC_B_WORDS + DC_B_TYPE]].inv_m;
            for (int q = 0; q < 3; ++q) { va[q] += dl * ima * w.d[q]; va[3 + q] += dl * w.ka[q]; }
            if (vb) {
                const R imb = A.t[(int)B[w.b * DC_B_WORDS + DC_B_TYPE]].inv_m;
                for (int q = 0; q < 3; ++q) { vb[q] -= dl * imb * w.d[q]; vb[3 + q] -= dl * w.kb[q]; }
            }
        }
    }
}

// semi-implicit Euler, quaternion q += dt/2 (w, 0) * q, renormalised
template <class R> DC_HD void dc_integrate(const DcScene<R>& S, R* B, int k) {
    R* b = B + k * DC_B_WORDS;
    if (b[DC_B_PRESENT] == (R)0) return;
    for (int r = 0; r < 3; ++r) b[DC_B_P + r] += S.dt * b[DC_B_V + r];
    const R wx = b[DC_B_W], wy = b[DC_B_W + 1], wz = b[DC_B_W + 2];
    R* q = b + DC_B_Q;
    const R h = (R)0.5 * S.dt;
    const R qx = q[0] + h * (wx * q[3] + wy * q[2] - wz * q[1]);
    const R qy = q[1] + h * (wy * q[3] + wz * q[0] - wx * q[2]);
    const R qz = q[2] + h * (wz * q[3] + wx * q[1] - wy * q[0]);
    const R qw = q[3] - h * (wx * q[0] + wy * q[1] + wz * q[2]);
    const R inv = (R)1 / sqrt(qx * qx + qy * qy + qz * qz + qw * qw);
    q[0] = qx * inv; q[1] = qy * inv; q[2] = qz * inv; q[3] = qw * inv;
}

// One micro-step of all bodies in one thread.  `arm` = DC_MAXARM x (cx, cy, cz, r) of the arm's collision spheres at the start of the
// micro-step (narm used); `kick` (nullable) = impulse on the sphere (slot 10) in this micro-step.  `rows` is scratch of 3 * DC_MAXC
// rows.  `touch` (nullable) accumulates body-body / arm contacts.
template <class R>
DC_HD void dc_step(const DcAssets<R>& A, const DcScene<R>& S, R* B, const R* arm, int narm, const R* kick, DcRow<R>* rows, DcTouch* touch) {
    DcWork<R> W;
    uint32_t adj[DC_NBODY];
    int root[DC_NBODY];
    for (int k = 0; k < DC_NBODY; ++k) dc_prepare(A, B, k, W, kick, S);
    for (int k = 0; k < DC_NBODY; ++k) adj[k] = dc_adjacency(A, S, B, W, k);
    dc_island_roots(adj, root);
    for (int r = 0; r < DC_NBODY; ++r)
        if (root[r] == r && B[r * DC_B_WORDS + DC_B_PRESENT] != (R)0) dc_island_solve(A, S, B, W, r, root, arm, narm, rows, touch);
    for (int k = 0; k < DC_NBODY; ++k) dc_integrate(S, B, k);
}

// the kick of step() at _env_step_counter == 10 (:117-125): horizontal unit direction from two normal draws, scaled to BALL_FORCE,
// z = 1, component-wise absolute value; applied for one micro-step -> impulse = force * dt
template <class R> DC_HD void dc_kick(double n0, double n1, R dt, R* imp) {
    const double l = sqrt(n0 * n0 + n1 * n1);
    const double fx = l > 0.0 ? fabs(n0 / l * DC_BALL_FORCE) : DC_BALL_FORCE, fy = l > 0.0 ? fabs(n1 / l * DC_BALL_FORCE) : 0.0;
    imp[0] = (R)fx * dt; imp[1] = (R)fy * dt; imp[2] = (R)1 * dt;
}
