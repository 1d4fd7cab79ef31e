/*
 * ORACLE (test infrastructure, not product code) -- the image path of include/srl_sim.h on the host: the CPU checker of the CUDA
 * library's frames.  Every entry point draws through render_frames: the same primitive lists (the oracle's env state in float32) and
 * per-pixel arithmetic (csrc/render_core.h) as the kernels, frames in host memory, no culling.
 */
#include <string.h>
#include <vector>
#include "oracle_sim.h"
#include "../robotics-rl-srl_b200/csrc/render_core.h"

/* Env i's frame through cams[i] (per_env) or cams[0].  With follow_robot (MobileRobot) the camera's target x, y are offsets from the
 * robot: float32(float64 position + float64 offset), z absolute.  With L, the env's scene list is followed by its bodies
 * B + i * DC_NBODY * DC_B_WORDS (srl_distractor_prims). */
static void render_frames(const srl_sim* s, const srl_camera* cams, bool per_env, int follow_robot, const SrlBodyLooks* L, const float* B,
                          int width, int height, uint8_t* rgb_out) {
    std::vector<SrlPrim> prims(SRL_MAX_PRIMS);
    std::vector<SrlPrep> prep(SRL_MAX_PRIMS);
    for (int i = 0; i < s->n; ++i) {
        const srl_camera& cam = cams[per_env ? i : 0];
        float target[3] = {cam.target[0], cam.target[1], cam.target[2]};
        int np;
        if (s->kuka) np = oracle_kuka_scene(s, i, prims.data());
        else {
            const MobileEnv& e = s->mobile[i];
            if (follow_robot) {
                target[0] = (float)(e.pos[0] + (double)target[0]);
                target[1] = (float)(e.pos[1] + (double)target[1]);
            }
            np = srl_mobile_scene(srl_mobile_render_kind(s->kind), (float)e.pos[0], (float)e.pos[1], (float)e.target[0][0], (float)e.target[0][1],
                                  (float)e.target[1][0], (float)e.target[1][1], prims.data());
        }
        if (L) np = srl_distractor_prims(*L, B + (size_t)i * DC_NBODY * DC_B_WORDS, np, prims.data());
        SrlCam c;
        srl_camera_setup(target, cam.distance, cam.yaw, cam.pitch, cam.roll, cam.fov, width, height, c);
        for (int k = 0; k < np; ++k) srl_prepare(c.eye, prims[k], prep[k]);
        uint8_t* frame = rgb_out + (size_t)i * height * width * 3;
        for (int y = 0; y < height; ++y)
            for (int x = 0; x < width; ++x)
                srl_render_pixel(c, prep.data(), prims.data(), srl_prim_mask_all(np), x, y, frame + ((size_t)y * width + x) * 3);
    }
}

extern "C" {

int srl_sim_render(srl_sim* s, const srl_camera* cam, int width, int height, uint8_t* rgb_out, void*) {
    if (!s || !cam || !rgb_out) { oracle_set_error("render: null argument"); return 1; }
    char msg[256];
    if (srl_render_args_error(false, s->kind, cam, 1, 0, width, height, msg, sizeof(msg))) { oracle_set_error("%s", msg); return 1; }
    render_frames(s, cam, false, 0, NULL, NULL, width, height, rgb_out);
    return 0;
}

int srl_sim_render_cameras(srl_sim* s, const srl_camera* cams, int follow_robot, int width, int height, uint8_t* rgb_out, void*) {
    if (!s || !cams || !rgb_out) { oracle_set_error("render_cameras: null argument"); return 1; }
    char msg[256];
    if (srl_render_args_error(true, s->kind, cams, s->n, follow_robot, width, height, msg, sizeof(msg))) { oracle_set_error("%s", msg); return 1; }
    render_frames(s, cams, true, follow_robot, NULL, NULL, width, height, rgb_out);
    return 0;
}

/* The CPU oracle has no distractor body dynamics (oracle_render_bodies below draws caller-given bodies instead): the entry point exists so
 * that both libraries export every symbol of include/srl_sim.h. */
int srl_sim_set_distractors(srl_sim*, const void*, size_t) {
    oracle_set_error("set_distractors: the CPU oracle has no distractor body dynamics");
    return 1;
}

} /* extern "C" */

/* Test hook: the frames of a KukaRandButton handle with caller-given bodies (typically SRL_F_DISTRACTORS of a CUDA handle), which stay where
 * they are put.  bodies = f64[N][DC_NBODY][9] (position, quaternion x y z w, type, present), drawn with the asset blob's drawing words.
 * Returns 0, or 1 with srl_sim_last_error(). */
extern "C" int oracle_render_bodies(srl_sim* s, const double* blob, size_t blob_bytes, const double* bodies, const srl_camera* cam, int width,
                                    int height, uint8_t* rgb_out) {
    if (!s || !blob || !bodies || !cam || !rgb_out) { oracle_set_error("render_bodies: null argument"); return 1; }
    if (s->kind != SRL_ENV_KUKA_RAND_BUTTON) { oracle_set_error("render_bodies: only KukaRandButtonGymEnv-v0 has distractor bodies"); return 1; }
    if (width <= 0 || height <= 0) { oracle_set_error("render_bodies: bad image size"); return 1; }
    if (const char* err = dc_blob_error(blob, blob_bytes)) { oracle_set_error("render_bodies: %s", err); return 1; }
    SrlBodyLooks L;
    srl_body_looks(blob, L);
    std::vector<float> B((size_t)s->n * DC_NBODY * DC_B_WORDS, 0.f);
    for (int i = 0; i < s->n; ++i)
        for (int k = 0; k < DC_NBODY; ++k) {
            const double* in = bodies + ((size_t)i * DC_NBODY + k) * 9;
            if (!(in[7] >= 0.0 && in[7] < DC_NTYPE && in[7] == (double)(int)in[7]) || !(in[8] == 0.0 || in[8] == 1.0)) {
                oracle_set_error("render_bodies: env %d body %d: type must be 0..3 and present 0 or 1", i, k);
                return 1;
            }
            float* b = B.data() + ((size_t)i * DC_NBODY + k) * DC_B_WORDS;
            for (int a = 0; a < 7; ++a) b[DC_B_P + a] = (float)in[a];
            b[DC_B_TYPE] = (float)in[7];
            b[DC_B_PRESENT] = (float)in[8];
        }
    render_frames(s, cam, false, 0, &L, B.data(), width, height, rgb_out);
    return 0;
}
