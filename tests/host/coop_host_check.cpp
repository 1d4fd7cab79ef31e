// Host check of csrc/kuka_coop.cuh (four lanes per env, phases through a scratch area) against the one-thread-per-env functions of
// csrc/kuka_device.cuh, both compiled for the CPU: the model filled by the library's kuka_params_from_blob (csrc/kuka_params.cuh), random
// joint states, with and without contacts.
// Test infrastructure.  Build + run: tests/test_coop_host_cpu.py (g++ -O1 -ffp-contract=off).  Usage: coop_host_check <blob.bin> [cases]
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
// ---- shims so that the device headers parse as plain C++ ----
#define __device__
#define __forceinline__ inline
struct uint4 { uint32_t x, y, z, w; };
static inline uint4 make_uint4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { uint4 r = {a, b, c, d}; return r; }
static inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
static inline double rsqrt(double x) { return 1.0 / sqrt(x); }
static inline float __saturatef(float x) { return x < 0.f ? 0.f : x > 1.f ? 1.f : x; }
#include "../../robotics-rl-srl_b200/csrc/kuka_device.cuh"
#include "../../robotics-rl-srl_b200/csrc/kuka_coop.cuh"

static double urand() { return rand() / (double)RAND_MAX; }
static double g_max_rel[16];
static void cmp(int slot, const char* what, double a, double b, double tol_abs, double tol_rel) {
    const double err = fabs(a - b), den = fabs(a) > fabs(b) ? fabs(a) : fabs(b);
    if (err / (den + 1e-30) > g_max_rel[slot] && err > tol_abs * 0.01) g_max_rel[slot] = err / (den + 1e-30);
    if (err > tol_abs + tol_rel * den) { printf("MISMATCH %s: %.9g vs %.9g (err %.3g)\n", what, a, b, err); exit(1); }
}

template <bool TWOB>
static void run_cases(const KukaParams& P0, int cases) {
    std::vector<float> store((size_t)KC_ROWS4 * 4 + 8, 0.f), tab(KC_CONST_WORDS, 0.f);
    int n_contact_cases = 0;
    for (int cs = 0; cs < cases; ++cs) {
        KukaParams P = P0;
        KukaEnv e; memset(&e, 0, sizeof(e));
        for (int i = 0; i < KK_NB; ++i) { e.q[i] = P.snap_q[i] + (float)(0.6 * (urand() - 0.5)); e.qd[i] = (float)(2.0 * (urand() - 0.5)); }
        e.qb = (float)(0.01 * urand()); e.qb2 = (float)(0.01 * urand());
        e.bbx = P.btn_base[0]; e.bby = P.btn_base[1]; e.bbz = P.btn_base[2]; e.bb2x = P.btn_base[0]; e.bb2y = -P.btn_base[1] - 0.25f;
        KukaKin k; KukaContacts ct; memset(&ct, 0, sizeof(ct));
        kuka_fk<TWOB>(P, e, k, ct);
        if (cs % 3) {
            // put the table / the button right under the lowest collision sphere so that the contact code runs
            float zlow = 1e30f; int blow = 0;
            for (int sidx = 0; sidx < P.nsph; ++sidx) { const int b = P.sph_body[sidx]; if (k.p[b].z < zlow) { zlow = k.p[b].z; blow = b; } }
            if (cs % 3 == 1) P.table_z = zlow - 0.03f - (float)(0.02 * urand());
            else { e.bbx = k.p[blow].x + (float)(0.02 * (urand() - 0.5)); e.bby = k.p[blow].y; e.bbz = zlow - 0.06f - P.glider_z - P.disc_z1 + (float)(0.02 * urand()); P.table_z = e.bbz - 0.5f; }
            kuka_fk<TWOB>(P, e, k, ct);
        }
        // ---- four-lane path ----
        kc_fill_const(P, tab.data(), 0, 1);
        KcScratch s; s.b = store.data();
        KcKinIn in; memset(&in, 0, sizeof(in));
        for (int i = 0; i < KK_NB; ++i) in.q[i] = e.q[i];
        in.qb = e.qb; in.qb2 = e.qb2; in.bbx = e.bbx; in.bby = e.bby; in.bbz = e.bbz; in.bb2x = e.bb2x; in.bb2y = e.bb2y;
        const bool near = kc_kinematics<TWOB>(s, tab.data(), P, in);
        for (int i = 0; i < KK_NB; ++i) {
            const int o = i * KC_BS;
            const float* kp[4] = {&k.p[i].x, &k.a[i].x, &k.c[i].x, &k.pv[i].x};
            const int off[4] = {KB_P, KB_A, KB_C, KB_PV};
            for (int f = 0; f < 4; ++f) for (int t = 0; t < 3; ++t) cmp(0, "kinematics p/a/c/pv", kp[f][t], s[o + off[f] + t], 2e-6, 1e-5);
            for (int t = 0; t < 6; ++t) cmp(1, "Iw", k.Iw[i][t], s[o + KB_IW + t], 1e-6, 1e-5);
        }
        for (int t = 0; t < 9; ++t) cmp(0, "R6", k.R6[t], s[6 * KC_BS + KB_R + t], 2e-6, 1e-5);
        for (int t = 0; t < 3; ++t) { cmp(0, "grip", e.grip[t], s[8 * KC_BS + KB_C + t], 2e-6, 1e-5); cmp(0, "eepos", e.eepos[t], s[6 * KC_BS + KB_P + t], 2e-6, 1e-5); }
        const int flags = near ? (int)s[KC_OFF_LINK + 6] : 0, nc = near ? (int)s[KC_OFF_LINK + 7] : 0;
        if ((flags & 1) != e.cbutton || ((flags >> 1) & 1) != e.ctable || nc != ct.n) {
            printf("MISMATCH flags/nc: button %d/%d table %d/%d nc %d/%d\n", flags & 1, e.cbutton, (flags >> 1) & 1, e.ctable, nc, ct.n); exit(1);
        }
        if (TWOB && ((((flags >> 2) & 1) != e.cany0) || (((flags >> 3) & 1) != e.cany1))) { printf("MISMATCH any-link flags\n"); exit(1); }
        n_contact_cases += nc > 0;
        for (int c = 0; c < nc; ++c) {
            const int o = KC_OFF_CT + c * KC_CTS;
            if ((int)s[o] != ct.body[c] || (int)s[o + 1] != ct.shape[c]) { printf("MISMATCH contact %d body/shape\n", c); exit(1); }
            cmp(2, "contact dist", ct.dist[c], s[o + 2], 3e-6, 1e-5);
            const float* nn = &ct.nrm[c].x; const float* pt = &ct.pt[c].x;
            for (int t = 0; t < 3; ++t) { cmp(2, "contact normal", nn[t], s[o + 3 + t], 1e-4, 1e-4); cmp(2, "contact point", pt[t], s[o + 6 + t], 3e-6, 1e-5); }
        }
        // ---- dynamics: M^-1 and bias ----
        float A[KK_NB][KK_NB], bias[KK_NB];
        kuka_dynamics(P, e, k, A, bias);
        float Mref[KK_NB][KK_NB];
        memcpy(Mref, A, sizeof(A));
        kuka_spd_inverse(A);
        // the four-lane path: mass matrix and bias through the scratch area; every lane then inverts M in registers with the same code
        kc_dynamics(s, P, e.qd);
        float Anew[KK_NB][KK_NB];
        for (int i = 0; i < KK_NB; ++i) {
            cmp(3, "bias", bias[i], s[KC_OFF_BIAS + i], 2e-4, 2e-4);
            for (int j = 0; j <= i; ++j) {
                cmp(6, "M", Mref[i][j], s[KC_OFF_MA + i * KC_MS + j], 2e-5 * sqrt(fabs((double)Mref[i][i] * Mref[j][j])), 0.0);
                Anew[i][j] = s[KC_OFF_MA + i * KC_MS + j];
            }
        }
        kuka_spd_inverse(Anew);
        for (int i = 0; i < KK_NB; ++i)
            for (int j = 0; j <= i; ++j) cmp(4, "M^-1", A[i][j], Anew[i][j], 5e-3 * sqrt(fabs((double)A[i][i] * A[j][j])), 0.0);
        // ---- contact rows against a plain restatement ----
        if (nc > 0) {
            KC_RUN((kc_ph_rows<TWOB, false>(s, P, Anew, nc, u)));
            for (int r = 0; r < 3 * nc; ++r) {
                const int ro = KC_OFF_ROWS + r * KC_RS;
                double D = 0;
                for (int i = 0; i < KK_NB; ++i) {
                    double w = 0;
                    for (int j = 0; j < KK_NB; ++j) w += (double)(i >= j ? Anew[i][j] : Anew[j][i]) * s[ro + j];
                    cmp(5, "row W", w, s[ro + KK_ROW_W + i], 1e-3 * (fabs(w) + sqrt(fabs((double)A[i][i]))), 0.0);
                    D += w * s[ro + i];
                }
                D += (double)s[ro + KK_NB] * s[ro + KK_NB] * P.btn_minv;
                if (TWOB) D += (double)s[ro + KK_NB + 1] * s[ro + KK_NB + 1] * P.btn_minv;
                cmp(5, "row 1/D", 1.0 / D, s[ro + KK_ROW_INVD], 0.0, 2e-3);
                if (r < nc) {
                    // the normal row's Jacobian: n . (a_j x (pt - p_j)) for the ancestors of the contact body
                    const int c = r, body = ct.body[c];
                    for (int j = 0; j < KK_NB; ++j) {
                        const bool anc = (j == body) || (j <= 7 && j < body) || (j == 8 && body == 9) || (j == 10 && body == 11);
                        const f3 lever = cross3(k.a[j], ct.pt[c] - k.p[j]);
                        cmp(5, "row J", anc ? dot3(ct.nrm[c], lever) : 0.f, s[ro + j], 1e-5, 1e-4);
                    }
                    const float pen = ct.dist[c];
                    cmp(5, "row target", pen > 0.f ? -pen * P.inv_dt : -P.erp * pen * P.inv_dt, s[ro + KK_ROW_TGT], 1e-3, 1e-4);
                }
            }
        }
    }
    printf("%s: %d cases ok (%d with contacts); max relative differences: kinematics %.2e, Iw %.2e, contacts %.2e, bias %.2e, M %.2e, M^-1 %.2e, rows %.2e\n",
           TWOB ? "two-button" : "one-button", cases, n_contact_cases, g_max_rel[0], g_max_rel[1], g_max_rel[2], g_max_rel[3], g_max_rel[6], g_max_rel[4], g_max_rel[5]);
    if (n_contact_cases < cases / 4) { printf("too few contact cases\n"); exit(1); }
}

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: coop_host_check <blob.bin> [cases]\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { printf("cannot open %s\n", argv[1]); return 2; }
    std::vector<double> blob(1 << 16);
    const size_t n = fread(blob.data(), sizeof(double), blob.size(), f);
    fclose(f);
    KukaParams P;   // the model part of the library's parameter block, at the blob's own time step
    if (const char* err = kuka_params_from_blob(blob.data(), n * sizeof(double), 0.0, P)) { printf("%s\n", err); return 2; }
    const int cases = argc > 2 ? atoi(argv[2]) : 300;
    srand(12345);
    run_cases<false>(P, cases);
    memset(g_max_rel, 0, sizeof(g_max_rel));
    run_cases<true>(P, cases);
    return 0;
}
