// CPU checker of srl_sim_render_cameras (include/srl_sim.h; test infrastructure).  The oracle library implements srl_sim_render with one
// camera for the batch; this adds the per-env-camera entry point over an oracle handle, with the same primitive lists and per-pixel
// arithmetic (render_core.h) and the same camera set-up per env: with follow_robot, target x, y = float32(float64 robot position +
// float64(offset)), z absolute.  Compiled by tests/render_cameras_ref.py against oracle/liboracle_sim.so; the library it makes resolves
// every other srl_sim_* symbol (and srl_sim_last_error, whose message oracle_set_error sets) from the oracle library.
#include <vector>
#include "../../oracle/oracle_sim.h"
#include "../../robotics-rl-srl_b200/csrc/render_core.h"

static bool is_mobile_kind(int kind) { return kind >= SRL_ENV_MOBILE && kind <= SRL_ENV_MOBILE_LINE_TARGET; }

extern "C" int srl_sim_render_cameras(srl_sim* s, const srl_camera* cams, int follow_robot, int width, int height, uint8_t* rgb_out, void*) {
    if (!s || !cams || !rgb_out) { oracle_set_error("render_cameras: null argument"); return 1; }
    if (width <= 0 || height <= 0 || width > 4096 || height > 4096) { oracle_set_error("render_cameras: bad image size %d x %d", width, height); return 1; }
    if (follow_robot && !is_mobile_kind(s->kind)) { oracle_set_error("render_cameras: follow_robot needs a MobileRobot env kind (got kind %d)", s->kind); return 1; }
    for (int i = 0; i < s->n; ++i)
        if (!(cams[i].distance > 0.f) || !(cams[i].fov > 0.f && cams[i].fov < 180.f)) {
            oracle_set_error("render_cameras: bad camera %d (distance %g, fov %g)", i, cams[i].distance, cams[i].fov);
            return 1;
        }
    std::vector<SrlPrim> prims(SRL_MAX_PRIMS);
    std::vector<SrlPrep> prep(SRL_MAX_PRIMS);
    const int rk = s->kind == SRL_ENV_MOBILE_2TARGET ? 1 : s->kind == SRL_ENV_MOBILE_LINE_TARGET ? 2 : s->kind == SRL_ENV_MOBILE_1D ? 3 : 0;
    for (int i = 0; i < s->n; ++i) {
        float target[3] = {cams[i].target[0], cams[i].target[1], cams[i].target[2]};
        int np;
        if (is_mobile_kind(s->kind)) {
            const MobileEnv& e = s->mobile[i];
            if (follow_robot) {
                target[0] = (float)(e.pos[0] + (double)target[0]);
                target[1] = (float)(e.pos[1] + (double)target[1]);
            }
            np = srl_mobile_scene(rk, (float)e.pos[0], (float)e.pos[1], (float)e.target[0][0], (float)e.target[0][1], (float)e.target[1][0],
                                  (float)e.target[1][1], prims.data());
        } else np = oracle_kuka_scene(s, i, prims.data());
        SrlCam c;
        srl_camera_setup(target, cams[i].distance, cams[i].yaw, cams[i].pitch, cams[i].roll, cams[i].fov, width, height, c);
        for (int k = 0; k < np; ++k) srl_prepare(c.eye, prims[k], prep[k]);
        uint8_t* frame = rgb_out + (size_t)i * height * width * 3;
        for (int y = 0; y < height; ++y)
            for (int x = 0; x < width; ++x)
                srl_render_pixel(c, prep.data(), prims.data(), srl_prim_mask_all(np), x, y, frame + ((size_t)y * width + x) * 3);
    }
    return 0;
}
