// CPU checker of KukaRandButton frames with distractor bodies (test infrastructure).  The CPU oracle has no body dynamics, so the bodies
// come from the caller -- typically SRL_F_DISTRACTORS of a CUDA handle -- and stay where they are put.  Each env's list is the oracle's
// scene list (oracle_kuka_scene) followed by the bodies through the builder the CUDA list kernel uses (render_core.h:
// srl_distractor_prims), drawn by the same per-pixel arithmetic as the oracle's srl_sim_render.  Compiled by tests/distractor_frames_ref.py
// against oracle/liboracle_sim.so.
#include <stdio.h>
#include <string.h>
#include <vector>
#include "../../oracle/oracle_sim.h"
#include "../../robotics-rl-srl_b200/csrc/render_core.h"

static char g_err[256] = "";

extern "C" {

const char* dfr_last_error(void) { return g_err; }

// One width x height frame per env of an oracle KukaRandButton handle with the bodies `bodies` (f64[N][DC_NBODY][9], the SRL_F_DISTRACTORS
// layout: position, quaternion x y z w, type, present) drawn by the asset blob's drawing words.  Returns 0, or 1 with dfr_last_error().
int dfr_render(srl_sim* s, const double* blob, size_t blob_bytes, const double* bodies, const srl_camera* cam, int width, int height,
               uint8_t* rgb_out) {
    if (!s || !blob || !bodies || !cam || !rgb_out) { snprintf(g_err, sizeof(g_err), "dfr_render: null argument"); return 1; }
    if (s->kind != SRL_ENV_KUKA_RAND_BUTTON) { snprintf(g_err, sizeof(g_err), "dfr_render: only KukaRandButtonGymEnv-v0 has distractor bodies"); return 1; }
    if (width <= 0 || height <= 0) { snprintf(g_err, sizeof(g_err), "dfr_render: bad image size"); return 1; }
    if (const char* err = dc_blob_error(blob, blob_bytes)) { snprintf(g_err, sizeof(g_err), "dfr_render: %s", err); return 1; }
    SrlBodyLooks L;
    srl_body_looks(blob, L);
    SrlCam c;
    srl_camera_setup(cam->target, cam->distance, cam->yaw, cam->pitch, cam->roll, cam->fov, width, height, c);
    std::vector<SrlPrim> prims(SRL_MAX_PRIMS);
    std::vector<SrlPrep> prep(SRL_MAX_PRIMS);
    float B[DC_NBODY * DC_B_WORDS];
    for (int i = 0; i < s->n; ++i) {
        memset(B, 0, sizeof(B));
        for (int k = 0; k < DC_NBODY; ++k) {
            const double* in = bodies + ((size_t)i * DC_NBODY + k) * 9;
            if (!(in[7] >= 0.0 && in[7] < DC_NTYPE && in[7] == (double)(int)in[7]) || !(in[8] == 0.0 || in[8] == 1.0)) {
                snprintf(g_err, sizeof(g_err), "dfr_render: env %d body %d: type must be 0..3 and present 0 or 1", i, k);
                return 1;
            }
            for (int a = 0; a < 7; ++a) B[k * DC_B_WORDS + DC_B_P + a] = (float)in[a];
            B[k * DC_B_WORDS + DC_B_TYPE] = (float)in[7];
            B[k * DC_B_WORDS + DC_B_PRESENT] = (float)in[8];
        }
        int np = oracle_kuka_scene(s, i, prims.data());
        np = srl_distractor_prims(L, B, np, prims.data());
        for (int k = 0; k < np; ++k) srl_prepare(c.eye, prims[k], prep[k]);
        uint8_t* frame = rgb_out + (size_t)i * height * width * 3;
        for (int y = 0; y < height; ++y)
            for (int x = 0; x < width; ++x)
                srl_render_pixel(c, prep.data(), prims.data(), srl_prim_mask_all(np), x, y, frame + ((size_t)y * width + x) * 3);
    }
    return 0;
}

}  // extern "C"
