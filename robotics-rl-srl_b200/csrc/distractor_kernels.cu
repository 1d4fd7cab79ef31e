// KukaRandButton's distractor bodies (opt-in, srl_sim_set_distractors; distractor_core.h) -- kernel and host side (sm_90a).  The arm never
// feels them, so after every traced kuka_kernel launch (kuka_kernels.cu) a kernel of their own replays the micro-steps it recorded.
#include <string.h>
#include <vector>
#include "common.cuh"
#include "kuka_state.cuh"
#include "kuka_device.cuh"
#include "distractor_core.h"
#include "render_core.h"

// Trace capacity: T (action_repeat + 5) micro-steps per env -- at 4096 envs x 128 steps x (1 + 5) that is 201 MB.  The arm's 500 settle
// micro-steps are one fixed trajectory per handle (`settle`).
struct DistDev {
    float* body;         // [N][DC_NBODY][DC_B_WORDS]
    uint32_t* touch;     // [N][2] bodies that touched another body / the arm since their placement (bit k = slot k)
    float4* trace;       // [cap][4][N]
    int* trace_len;      // [N] micro-steps of the last traced launch
    float4* settle;      // [500][4] the arm's settle trajectory
    size_t cap;          // micro-steps per env the trace holds
    DcAssets<float> A;
};
// The host's view of a handle's bodies: DistDev (distractor_kernel's parameter, unchanged) plus the per-type drawing table that
// srl_sim_render's list kernel reads.
struct DistHost : DistDev {
    SrlBodyLooks looks;
};

namespace {

// Philox purposes of the bodies (philox.cuh: 0-10 are the simulator's, policy_core.h: 16 and up the policy's): 0x100-0x109 placement k,
// 0x10A kick direction, 0x10B-0x10D object types
enum { PHILOX_PURPOSE_DIST_PLACE = 0x100, PHILOX_PURPOSE_DIST_KICK = 0x10A, PHILOX_PURPOSE_DIST_TYPE = 0x10B /* 0x10B-0x10D */ };

// world centres and radii of the arm's collision spheres at joint configuration q
KK_DEV int arm_spheres(const KukaParams& P, const float* q, float* out) {
    float Rb[KK_NB][9]; f3 pb[KK_NB];
    kuka_world_frames(P, q, Rb, pb);
    const int ns = P.nsph < DC_MAXARM ? P.nsph : DC_MAXARM;
    for (int k = 0; k < ns; ++k) {
        const int b = P.sph_body[k];
        const float* Rk = Rb[b];
        out[4 * k] = pb[b].x + Rk[0] * P.sph_c[k][0] + Rk[1] * P.sph_c[k][1] + Rk[2] * P.sph_c[k][2];
        out[4 * k + 1] = pb[b].y + Rk[3] * P.sph_c[k][0] + Rk[4] * P.sph_c[k][1] + Rk[5] * P.sph_c[k][2];
        out[4 * k + 2] = pb[b].z + Rk[6] * P.sph_c[k][0] + Rk[7] * P.sph_c[k][1] + Rk[8] * P.sph_c[k][2];
        out[4 * k + 3] = P.sph_r[k];
    }
    return ns;
}

// the scene of one micro-step from a trace record: button base + disc at the glider q
KK_DEV void dist_scene(const KukaParams& P, DcScene<float>& S, float qb, float bx, float by) {
    S.bx = bx; S.by = by; S.bz = P.btn_base[2];
    S.disc0 = S.bz + P.glider_z + qb + P.disc_z0; S.disc1 = S.bz + P.glider_z + qb + P.disc_z1;
}

// A group of 16 lanes per env (2 envs per warp) advances its bodies through the micro-steps the preceding traced kuka_kernel launch
// recorded: lane k < 11 owns body k (prepare, adjacency, integrate), and the lowest lane of every island of bodies in contact runs that
// island's rows and sweeps (distractor_core.h: the same arithmetic as the one-thread dc_step).  Body state and the per-micro-step work
// arrays live in shared memory; a lane's contact rows in its own local memory.  At the first micro-step of a reset() the group places the
// bodies (host values or the env's counter-based stream) and runs the 500 settle micro-steps against the arm's settle trajectory first.
constexpr int DIST_LANES = 16, DIST_BLOCK = 128, DIST_ENVS_PER_BLOCK = DIST_BLOCK / DIST_LANES;
struct DistShared {
    float B[DC_NBODY * DC_B_WORDS];
    DcWork<float> W;
    uint32_t adj[DC_NBODY];
};

KK_DEV void dist_micro_step(const DcAssets<float>& A, const DcScene<float>& S, DistShared& sh, int u, unsigned gmask, const float* arm, int na,
                            const float* kick, DcRow<float>* rows, DcTouch& touch) {
    if (u < DC_NBODY) dc_prepare(A, sh.B, u, sh.W, kick, S);
    __syncwarp(gmask);
    if (u < DC_NBODY) sh.adj[u] = dc_adjacency(A, S, sh.B, sh.W, u);
    __syncwarp(gmask);
    int root[DC_NBODY];
    uint32_t adj[DC_NBODY];
    for (int k = 0; k < DC_NBODY; ++k) adj[k] = sh.adj[k];
    dc_island_roots(adj, root);
    if (u < DC_NBODY && root[u] == u && sh.B[u * DC_B_WORDS + DC_B_PRESENT] != 0.f) dc_island_solve(A, S, sh.B, sh.W, u, root, arm, na, rows, &touch);
    __syncwarp(gmask);
    if (u < DC_NBODY) dc_integrate(S, sh.B, u);
    __syncwarp(gmask);
}

__global__ void __launch_bounds__(DIST_BLOCK) distractor_kernel(const __grid_constant__ KukaDev d, const __grid_constant__ DistDev g, int n,
                                                                 const double* __restrict__ draws) {
    __shared__ DistShared shared[DIST_ENVS_PER_BLOCK];
    const int lane = threadIdx.x & 31, u = lane & (DIST_LANES - 1);
    const unsigned gmask = 0xFFFFu << (lane & ~(DIST_LANES - 1));
    const int slot = threadIdx.x / DIST_LANES;
    const int i = blockIdx.x * DIST_ENVS_PER_BLOCK + slot;
    if (i >= n) return;                      // whole groups leave together
    const int len = g.trace_len[i];
    if (len <= 0) return;
    DistShared& sh = shared[slot];
    const KukaParams& P = d.P;
    const size_t N = (size_t)n;
    const uint64_t genv = P.env_offset + (uint64_t)i;
    float* const gb = g.body + (size_t)i * DC_NBODY * DC_B_WORDS;
    for (int j = u; j < DC_NBODY * DC_B_WORDS; j += DIST_LANES) sh.B[j] = gb[j];
    DcTouch touch = {0u, 0u};
    DcScene<float> S;
    S.table_z = P.table_z; S.txmin = P.txmin; S.txmax = P.txmax; S.tymin = P.tymin; S.tymax = P.tymax;
    S.stack_top = P.stack_top; S.stack_r = P.stack_r; S.disc_r = P.disc_r;
    S.dt = P.dt; S.g = 10.f; S.margin = P.cdist; S.iters = P.iters;   // setGravity(0, 0, -10) (:71)
    DcRow<float> rows[3 * DC_MAXC];
    float arm[DC_MAXARM * 4];
    uint32_t clear = 0u;                     // lane 0: the touch masks were reset by a placement in this launch
    __syncwarp(gmask);
    for (int m = 0; m < len; ++m) {
        const size_t base = (size_t)m * 4 * N + (size_t)i;
        const float4 r0 = g.trace[base], r1 = g.trace[base + N], r2 = g.trace[base + 2 * N], r3 = g.trace[base + 3 * N];
        const int tag = __float_as_int(r3.w);
        const uint32_t episode = (uint32_t)tag >> 4;
        if (tag & DT_FIRST) {
            if (u == 0) {
                double xy[20]; int type[10];
                if ((tag & DT_HOST_DRAWS) && draws) {
                    const double* dr = draws + (size_t)i * KUKA_DIST_DRAWS;
                    for (int k = 0; k < 20; ++k) xy[k] = dr[18 + k];
                    for (int k = 0; k < 10; ++k) type[k] = (int)dr[38 + k];
                } else {
                    // x = 0.5 + 0.15 U(-1, 1), y = 0 + 0.3 U(-1, 1) (kuka_rand_button_gym_env.py:63-64); the object type from the same stream
                    for (int k = 0; k < 10; ++k) {
                        const uint4 r = philox4x32_10(P.seed, genv, episode, PHILOX_PURPOSE_DIST_PLACE + k);
                        xy[2 * k] = 0.5 + 0.15 * (-1.0 + 2.0 * philox_u01(r.x, r.y));
                        xy[2 * k + 1] = 0.3 * (-1.0 + 2.0 * philox_u01(r.z, r.w));
                    }
                    for (int k = 0; k < 10; k += 4) {
                        const uint4 r = philox4x32_10(P.seed, genv, episode, PHILOX_PURPOSE_DIST_TYPE + k / 4);
                        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
                        for (int j = 0; j < 4 && k + j < 10; ++j) type[k + j] = (int)__umulhi(w[j], 3u);   // randint(3)
                    }
                }
                dc_place(sh.B, xy, type, (double)r3.y, (double)r3.z);
            }
            touch.body = 0u; touch.arm = 0u; clear = 1u;
            __syncwarp(gmask);
            for (int s2 = 0; s2 < 500; ++s2) {    // p.stepSimulation() x 500 of reset() (:242-247), the arm on its settle trajectory
                const float4 a0 = __ldg(g.settle + 4 * s2), a1 = __ldg(g.settle + 4 * s2 + 1), a2 = __ldg(g.settle + 4 * s2 + 2), a3 = __ldg(g.settle + 4 * s2 + 3);
                const float q[KK_NB] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w};
                const int na = arm_spheres(P, q, arm);
                dist_scene(P, S, a3.x, r3.y, r3.z);
                dist_micro_step(g.A, S, sh, u, gmask, arm, na, nullptr, rows, touch);
            }
        }
        const float q[KK_NB] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w, r2.x, r2.y, r2.z, r2.w};
        const int na = arm_spheres(P, q, arm);
        dist_scene(P, S, r3.x, r3.y, r3.z);
        float imp[3];
        const bool kick = (tag & DT_KICK) != 0;
        if (kick) {
            // np.random.normal(size=(3,)), z dropped (:119-121): two normals of the env's stream
            const uint4 r = philox4x32_10(P.seed, genv, episode, PHILOX_PURPOSE_DIST_KICK);
            const double u1 = philox_u01(r.x, r.y), u2 = philox_u01(r.z, r.w);
            const double rad = sqrt(-2.0 * log(1.0 - u1));
            dc_kick(rad * cos(6.283185307179586 * u2), rad * sin(6.283185307179586 * u2), S.dt, imp);
        }
        dist_micro_step(g.A, S, sh, u, gmask, arm, na, kick ? imp : (const float*)nullptr, rows, touch);
    }
    for (int j = u; j < DC_NBODY * DC_B_WORDS; j += DIST_LANES) gb[j] = sh.B[j];
    // the group's touch masks: OR over the lanes, on top of the stored ones unless a placement cleared them
    for (int off = DIST_LANES / 2; off > 0; off >>= 1) {
        touch.body |= __shfl_xor_sync(gmask, touch.body, off);
        touch.arm |= __shfl_xor_sync(gmask, touch.arm, off);
    }
    if (u == 0) {
        if (!clear) { touch.body |= g.touch[2 * i]; touch.arm |= g.touch[2 * i + 1]; }
        g.touch[2 * i] = touch.body; g.touch[2 * i + 1] = touch.arm;
    }
}

}  // namespace

int dist_alloc(srl_sim* s, const void* blob, size_t bytes, float4** settle) {
    if (s->kind != SRL_ENV_KUKA_RAND_BUTTON) { srl_set_error("set_distractors: only KukaRandButtonGymEnv-v0 has distractor bodies"); return 1; }
    if (s->kuka_started) { srl_set_error("set_distractors: must be called between srl_sim_create and the first reset"); return 1; }
    if (s->kuka_next) { srl_set_error("set_distractors: not available together with srl_cfg.prefetch_resets"); return 1; }
    if (s->dist) { srl_set_error("set_distractors: already set"); return 1; }
    if (!blob) { srl_set_error("set_distractors: null asset blob"); return 1; }
    if (const char* err = dc_blob_error((const double*)blob, bytes)) { srl_set_error("set_distractors: %s", err); return 1; }
    DistHost* g = new DistHost();
    memset(g, 0, sizeof(*g));
    s->dist = g;   // freed by kuka_free, also when srl_sim_set_distractors fails after this point
    dc_assets_from_blob((const double*)blob, g->A);
    srl_body_looks((const double*)blob, g->looks);
    const size_t N = (size_t)s->n;
    SRL_CUDA_OK(cudaMalloc(&g->body, N * DC_NBODY * DC_B_WORDS * sizeof(float))); SRL_CUDA_OK(cudaMemset(g->body, 0, N * DC_NBODY * DC_B_WORDS * sizeof(float)));
    SRL_CUDA_OK(cudaMalloc(&g->touch, N * 2 * sizeof(uint32_t))); SRL_CUDA_OK(cudaMemset(g->touch, 0, N * 2 * sizeof(uint32_t)));
    SRL_CUDA_OK(cudaMalloc(&g->trace_len, N * sizeof(int))); SRL_CUDA_OK(cudaMemset(g->trace_len, 0, N * sizeof(int)));
    SRL_CUDA_OK(cudaMalloc(&g->settle, 500 * 4 * sizeof(float4)));
    *settle = g->settle;
    return 0;
}

int dist_trace(srl_sim* s, size_t steps, cudaStream_t st, float4** trace, int** trace_len) {
    DistDev* g = s->dist;
    const size_t N = (size_t)s->n;
    if (steps > g->cap) {
        SRL_CUDA_OK(cudaStreamSynchronize(st));
        cudaFree(g->trace); g->trace = nullptr; g->cap = 0;
        SRL_CUDA_OK(cudaMalloc(&g->trace, steps * 4 * N * sizeof(float4)));
        g->cap = steps;
    }
    SRL_CUDA_OK(cudaMemsetAsync(g->trace_len, 0, N * sizeof(int), st));
    *trace = g->trace; *trace_len = g->trace_len;
    return 0;
}

int dist_advance(srl_sim* s, const double* draws, cudaStream_t st) {
    distractor_kernel<<<(s->n + DIST_ENVS_PER_BLOCK - 1) / DIST_ENVS_PER_BLOCK, DIST_BLOCK, 0, st>>>(*s->kuka, *s->dist, s->n, draws);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

void dist_free(srl_sim* s) {
    if (DistDev* g = s->dist) {
        cudaFree(g->body); cudaFree(g->touch); cudaFree(g->trace); cudaFree(g->trace_len); cudaFree(g->settle);
        delete static_cast<DistHost*>(g);
        s->dist = nullptr;
    }
}

const float* dist_render_bodies(const srl_sim* s, SrlBodyLooks* looks) {
    if (!s->dist) return nullptr;
    *looks = static_cast<const DistHost*>(s->dist)->looks;
    return s->dist->body;
}

// SRL_F_DISTRACTORS and SRL_F_DISTRACTOR_TOUCH of kuka_get_state: zeros for a handle without bodies.  The test hooks (SRL_F_DISTRACTOR_RECORDS,
// _TRACE_LEN, _TRACE, _SETTLE) are plain copies of the device buffers and need the bodies.
int dist_get_state(srl_sim* s, int field, void* dst, size_t bytes) {
    const size_t N = (size_t)s->n;
    const DistDev* g = s->dist;
    if (field == SRL_F_DISTRACTORS || field == SRL_F_DISTRACTOR_TOUCH) {
        const bool touch = field == SRL_F_DISTRACTOR_TOUCH;
        if (bytes != (touch ? N * 2 * sizeof(uint32_t) : N * DC_NBODY * 9 * sizeof(double))) { srl_set_error("get_state: size mismatch"); return 1; }
        memset(dst, 0, bytes);
        if (!g) return 0;
        if (touch) { SRL_CUDA_OK(cudaMemcpy(dst, g->touch, bytes, cudaMemcpyDeviceToHost)); return 0; }
        std::vector<float> h(N * DC_NBODY * DC_B_WORDS);
        SRL_CUDA_OK(cudaMemcpy(h.data(), g->body, h.size() * sizeof(float), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < N * DC_NBODY; ++i) {
            const float* b = h.data() + i * DC_B_WORDS;
            double* o = (double*)dst + i * 9;
            for (int a = 0; a < 7; ++a) o[a] = b[DC_B_P + a];   // position, quaternion (x y z w)
            o[7] = b[DC_B_TYPE]; o[8] = b[DC_B_PRESENT];
        }
        return 0;
    }
    if (!g) { srl_set_error("get_state: field %d needs srl_sim_set_distractors", field); return 1; }
    switch (field) {
    case SRL_F_DISTRACTOR_RECORDS:
        if (bytes != N * DC_NBODY * DC_B_WORDS * sizeof(float)) { srl_set_error("get_state: size mismatch"); return 1; }
        SRL_CUDA_OK(cudaMemcpy(dst, g->body, bytes, cudaMemcpyDeviceToHost));
        return 0;
    case SRL_F_DISTRACTOR_TRACE_LEN:
        if (bytes != N * sizeof(int)) { srl_set_error("get_state: size mismatch"); return 1; }
        SRL_CUDA_OK(cudaMemcpy(dst, g->trace_len, bytes, cudaMemcpyDeviceToHost));
        return 0;
    case SRL_F_DISTRACTOR_SETTLE:
        if (bytes != 500 * 4 * sizeof(float4)) { srl_set_error("get_state: size mismatch"); return 1; }
        SRL_CUDA_OK(cudaMemcpy(dst, g->settle, bytes, cudaMemcpyDeviceToHost));
        return 0;
    case SRL_F_DISTRACTOR_TRACE: {
        const size_t L = bytes / (N * 4 * sizeof(float4));
        if (L == 0 || L > g->cap || bytes != L * N * 4 * sizeof(float4)) { srl_set_error("get_state: the trace holds %zu records per env", g->cap); return 1; }
        std::vector<float4> h(L * 4 * N);     // [micro-step][4][N] on the device -> [N][micro-step][4]
        SRL_CUDA_OK(cudaMemcpy(h.data(), g->trace, h.size() * sizeof(float4), cudaMemcpyDeviceToHost));
        float4* o = (float4*)dst;
        for (size_t i = 0; i < N; ++i)
            for (size_t m = 0; m < L; ++m)
                for (size_t r = 0; r < 4; ++r) o[(i * L + m) * 4 + r] = h[(m * 4 + r) * N + i];
        return 0;
    }
    default:
        srl_set_error("get_state: unknown field %d", field);
        return 1;
    }
}

// SRL_F_DISTRACTOR_RECORDS of kuka_set_state (test hook): valid records only
int dist_set_state(srl_sim* s, const void* src, size_t bytes) {
    const size_t N = (size_t)s->n;
    DistDev* g = s->dist;
    if (!g) { srl_set_error("set_state: the distractor records need srl_sim_set_distractors"); return 1; }
    if (bytes != N * DC_NBODY * DC_B_WORDS * sizeof(float)) { srl_set_error("set_state: size mismatch"); return 1; }
    for (size_t i = 0; i < N * DC_NBODY; ++i) {
        const float* b = (const float*)src + i * DC_B_WORDS;
        for (int a = 0; a < DC_B_WORDS; ++a)
            if (!isfinite(b[a])) { srl_set_error("set_state: distractor record %zu has a non-finite value", i); return 1; }
        if (b[DC_B_PRESENT] != 0.f && b[DC_B_PRESENT] != 1.f) { srl_set_error("set_state: distractor record %zu: present must be 0 or 1", i); return 1; }
        if (!(b[DC_B_TYPE] == 0.f || b[DC_B_TYPE] == 1.f || b[DC_B_TYPE] == 2.f || b[DC_B_TYPE] == 3.f)) { srl_set_error("set_state: distractor record %zu: type must be 0, 1, 2 or 3", i); return 1; }
        const double qq = (double)b[DC_B_Q] * b[DC_B_Q] + (double)b[DC_B_Q + 1] * b[DC_B_Q + 1] + (double)b[DC_B_Q + 2] * b[DC_B_Q + 2] + (double)b[DC_B_Q + 3] * b[DC_B_Q + 3];
        if (fabs(sqrt(qq) - 1.0) > 1e-4) { srl_set_error("set_state: distractor record %zu: the quaternion is not of unit length", i); return 1; }
    }
    SRL_CUDA_OK(cudaMemcpy(g->body, src, bytes, cudaMemcpyHostToDevice));
    return 0;
}
