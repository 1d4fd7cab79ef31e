// Image observations (SURVEY.md 8(f).4): per-pixel arithmetic of the batched ray-caster, shared by the sm_90a kernels
// (csrc/render_kernels.cu) and the CPU checker (oracle/oracle_render.cpp, test infrastructure).
//
// What the reference does: `render(mode='rgb_array')` asks PyBullet's TinyRenderer for a 224 x 224 frame of the scene through
// computeViewMatrixFromYawPitchRoll / computeProjectionMatrixFOV / getCameraImage (environments/kuka_gym/kuka_button_gym_env.py:370-420,
// environments/mobile_robot/mobile_robot_env.py:287-334), and `srl_model="raw_pixels"` returns that frame as the observation.
// What this is: a ray-caster of ANALYTIC primitives -- plane, sphere, capsule, upright cylinder, yaw-rotated box, fully rotated box -- with ambient +
// Lambert shading, through the same pinhole camera.  The meshes and textures TinyRenderer draws (pybullet_data: kuka_iiwa/meshes, table,
// racecar, plane checker) are absent from the reference checkout and from this image, so the arm is drawn as capsules between its joint
// frames plus its collision spheres, the table / walls as boxes, the buttons / targets as the z-extruded discs their collada meshes are:
// same camera, same layout, same colours where the reference's own URDFs give them (urdf/wall.urdf, urdf/cylinder.urdf,
// urdf/simple_button.urdf), but NOT TinyRenderer's pixels -- parity with reference frames is unpinned and cannot be pinned offline.
#pragma once
#include <math.h>
#include <stdint.h>
#include "distractor_core.h"

#if defined(__CUDACC__)
#define SRL_RHD __host__ __device__ __forceinline__
#else
#define SRL_RHD inline
#endif

#define SRL_PRIM_WORDS 16
#define SRL_MAX_PRIMS 48
enum { SRL_PRIM_PLANE = 0, SRL_PRIM_SPHERE = 1, SRL_PRIM_CAPSULE = 2, SRL_PRIM_CYL = 3, SRL_PRIM_BOX = 4, SRL_PRIM_OBOX = 5 };
// the single-button Kuka scene (plane, table, 4 legs, 2 button, 8 arm capsules, 4 gripper capsules, 11 gripper spheres) plus every
// distractor body of KukaRandButton must fit one list
#define SRL_KUKA_ONE_BUTTON_PRIMS 31
static_assert(SRL_KUKA_ONE_BUTTON_PRIMS + DC_NBODY <= SRL_MAX_PRIMS, "a KukaRandButton scene with all its bodies must fit SRL_MAX_PRIMS");

// One primitive = 16 floats: type, 11 geometry words, r g b, pad.
//   PLANE   a0 = z, a1 = checker period (0: plain), a2..4 = second colour of the checker
//   SPHERE  a0..2 centre, a3 radius
//   CAPSULE a0..2 end 0, a3..5 end 1, a6 radius
//   CYL     a0 cx, a1 cy, a2 z0, a3 z1, a4 radius            (upright, capped)
//   BOX     a0..2 centre, a3..5 half extents, a6 cos, a7 sin  (rotated about z)
//   OBOX    a0..2 centre, a3..5 half extents, a6..9 unit quaternion x y z w (any rotation; q and -q draw the same bytes)
struct SrlPrim { float type, a[11], r, g, b, pad; };

// pixel (x, y) (row 0 = top) looks along fwd + u right + v up with u = ub + su (x + 0.5), v = vb - sv (y + 0.5)
struct SrlCam { float eye[3], fwd[3], right[3], up[3], ub, su, vb, sv; };

SRL_RHD void srl_prim_set(SrlPrim& p, int type, float r, float g, float b) {
    p.type = (float)type; p.r = r; p.g = g; p.b = b; p.pad = 0.f;
    for (int i = 0; i < 11; ++i) p.a[i] = 0.f;
}
SRL_RHD void srl_prim_capsule(SrlPrim& p, const float* e0, const float* e1, float rad, float r, float g, float b) {
    srl_prim_set(p, SRL_PRIM_CAPSULE, r, g, b);
    for (int i = 0; i < 3; ++i) { p.a[i] = e0[i]; p.a[3 + i] = e1[i]; }
    p.a[6] = rad;
}
SRL_RHD void srl_prim_sphere(SrlPrim& p, const float* c, float rad, float r, float g, float b) {
    srl_prim_set(p, SRL_PRIM_SPHERE, r, g, b);
    for (int i = 0; i < 3; ++i) p.a[i] = c[i];
    p.a[3] = rad;
}
SRL_RHD void srl_prim_cyl(SrlPrim& p, float cx, float cy, float z0, float z1, float rad, float r, float g, float b) {
    srl_prim_set(p, SRL_PRIM_CYL, r, g, b);
    p.a[0] = cx; p.a[1] = cy; p.a[2] = z0; p.a[3] = z1; p.a[4] = rad;
}
SRL_RHD void srl_prim_box(SrlPrim& p, float cx, float cy, float cz, float hx, float hy, float hz, float yaw_cos, float yaw_sin, float r, float g, float b) {
    srl_prim_set(p, SRL_PRIM_BOX, r, g, b);
    p.a[0] = cx; p.a[1] = cy; p.a[2] = cz; p.a[3] = hx; p.a[4] = hy; p.a[5] = hz; p.a[6] = yaw_cos; p.a[7] = yaw_sin;
}
SRL_RHD void srl_prim_obox(SrlPrim& p, const float* c, const float* half, const float* quat, float r, float g, float b) {
    srl_prim_set(p, SRL_PRIM_OBOX, r, g, b);
    for (int i = 0; i < 3; ++i) { p.a[i] = c[i]; p.a[3 + i] = half[i]; }
    for (int i = 0; i < 4; ++i) p.a[6 + i] = quat[i];
}
SRL_RHD void srl_prim_plane(SrlPrim& p, float z, float checker, float r, float g, float b) {
    srl_prim_set(p, SRL_PRIM_PLANE, r, g, b);
    p.a[0] = z; p.a[1] = checker; p.a[2] = 0.68f; p.a[3] = 0.77f; p.a[4] = 0.93f;     // plane.urdf's checker is white / light blue (imgs/kuka.gif, imgs/mobile_robot.gif)
}

// ---- camera: pybullet's computeViewMatrixFromYawPitchRoll (upAxisIndex = 2) + computeProjectionMatrixFOV, as eye + basis (RECALLED from
//      PhysicsClientC_API.cpp: eye = target + Rz(yaw) Ry(roll) Rx(pitch) (0, -distance, 0), up = the same rotation of (0, 0, 1)) ----
// It is built in two parts.  The angle part (the trigonometry) runs on the host only.  The target part runs on the host, and on the device
// for cameras whose target follows the robot (srl_sim_render_cameras): it is written in explicitly rounded operations -- no FMA contraction,
// IEEE square root and division on both sides -- so that a camera finished on the device has the bits the host gives it.
struct SrlCamAngles { float R[9], distance, ub, su, vb, sv; };   // R = Rz(yaw) Ry(roll) Rx(pitch); ub..sv as in SrlCam
// a camera whose target is the robot's position plus off (x, y; z absolute), finished on the device
struct SrlCamFollow { SrlCamAngles a; float off[3]; };

SRL_RHD float srl_mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
SRL_RHD float srl_add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
SRL_RHD float srl_sub_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
SRL_RHD float srl_div_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
SRL_RHD float srl_sqrt_rn(float a) {
#if defined(__CUDA_ARCH__)
    return __fsqrt_rn(a);
#else
    return sqrtf(a);
#endif
}

SRL_RHD void srl_camera_angles(float distance, float yaw_deg, float pitch_deg, float roll_deg, float fov_deg, int W, int H, SrlCamAngles& a) {
    const float d2r = 0.01745329251994329547f;
    const float cy = cosf(yaw_deg * d2r), sy = sinf(yaw_deg * d2r), cp = cosf(pitch_deg * d2r), sp = sinf(pitch_deg * d2r);
    const float cr = cosf(roll_deg * d2r), sr = sinf(roll_deg * d2r);
    const float R[9] = {cy * cr, cy * sr * sp - sy * cp, cy * sr * cp + sy * sp,
                        sy * cr, sy * sr * sp + cy * cp, sy * sr * cp - cy * sp,
                        -sr, cr * sp, cr * cp};
    for (int i = 0; i < 9; ++i) a.R[i] = R[i];
    a.distance = distance;
    const float th = tanf(0.5f * fov_deg * d2r), aspect = (float)W / (float)H;      // computeProjectionMatrixFOV: vertical fov, aspect = width / height
    a.ub = -th * aspect; a.su = 2.f * th * aspect / (float)W;
    a.vb = th; a.sv = 2.f * th / (float)H;
}

SRL_RHD void srl_camera_target(const float* target, const SrlCamAngles& a, SrlCam& c) {
    const float* R = a.R;
    const float e[3] = {0.f, -a.distance, 0.f};
    float up0[3], f[3];
    for (int i = 0; i < 3; ++i) {
        c.eye[i] = srl_add_rn(srl_add_rn(srl_add_rn(target[i], srl_mul_rn(R[3 * i], e[0])), srl_mul_rn(R[3 * i + 1], e[1])), srl_mul_rn(R[3 * i + 2], e[2]));
        up0[i] = R[3 * i + 2];
        f[i] = srl_sub_rn(target[i], c.eye[i]);
    }
    const float fl = srl_sqrt_rn(srl_add_rn(srl_add_rn(srl_mul_rn(f[0], f[0]), srl_mul_rn(f[1], f[1])), srl_mul_rn(f[2], f[2])));
    for (int i = 0; i < 3; ++i) c.fwd[i] = srl_div_rn(f[i], fl);
    // right = fwd x up0, up = right x fwd (the lookAt basis of b3ComputeViewMatrixFromPositions)
    const float s[3] = {srl_sub_rn(srl_mul_rn(c.fwd[1], up0[2]), srl_mul_rn(c.fwd[2], up0[1])),
                        srl_sub_rn(srl_mul_rn(c.fwd[2], up0[0]), srl_mul_rn(c.fwd[0], up0[2])),
                        srl_sub_rn(srl_mul_rn(c.fwd[0], up0[1]), srl_mul_rn(c.fwd[1], up0[0]))};
    const float sl = srl_sqrt_rn(srl_add_rn(srl_add_rn(srl_mul_rn(s[0], s[0]), srl_mul_rn(s[1], s[1])), srl_mul_rn(s[2], s[2])));
    for (int i = 0; i < 3; ++i) c.right[i] = srl_div_rn(s[i], sl);
    c.up[0] = srl_sub_rn(srl_mul_rn(c.right[1], c.fwd[2]), srl_mul_rn(c.right[2], c.fwd[1]));
    c.up[1] = srl_sub_rn(srl_mul_rn(c.right[2], c.fwd[0]), srl_mul_rn(c.right[0], c.fwd[2]));
    c.up[2] = srl_sub_rn(srl_mul_rn(c.right[0], c.fwd[1]), srl_mul_rn(c.right[1], c.fwd[0]));
    c.ub = a.ub; c.su = a.su; c.vb = a.vb; c.sv = a.sv;
}

SRL_RHD void srl_camera_setup(const float* target, float distance, float yaw_deg, float pitch_deg, float roll_deg, float fov_deg, int W, int H, SrlCam& c) {
    SrlCamAngles a;
    srl_camera_angles(distance, yaw_deg, pitch_deg, roll_deg, fov_deg, W, H, a);
    srl_camera_target(target, a, c);
}

// ---- rotation by a unit quaternion q = (x y z w) and by its inverse, v' = v + w t + u x t with u = (x y z), t = 2 u x v (for the inverse
//      u -> -u).  Every product pairs two components of q, so q and -q give the same bits.
SRL_RHD void srl_quat_rotate(const float* q, const float* v, float* o) {
    const float t[3] = {2.f * (q[1] * v[2] - q[2] * v[1]), 2.f * (q[2] * v[0] - q[0] * v[2]), 2.f * (q[0] * v[1] - q[1] * v[0])};
    o[0] = v[0] + q[3] * t[0] + (q[1] * t[2] - q[2] * t[1]);
    o[1] = v[1] + q[3] * t[1] + (q[2] * t[0] - q[0] * t[2]);
    o[2] = v[2] + q[3] * t[2] + (q[0] * t[1] - q[1] * t[0]);
}
SRL_RHD void srl_quat_rotate_inv(const float* q, const float* v, float* o) {
    const float t[3] = {2.f * (v[1] * q[2] - v[2] * q[1]), 2.f * (v[2] * q[0] - v[0] * q[2]), 2.f * (v[0] * q[1] - v[1] * q[0])};
    o[0] = v[0] + q[3] * t[0] + (t[1] * q[2] - t[2] * q[1]);
    o[1] = v[1] + q[3] * t[1] + (t[2] * q[0] - t[0] * q[2]);
    o[2] = v[2] + q[3] * t[2] + (t[0] * q[1] - t[1] * q[0]);
}

// ---- per-camera prepared form of a primitive: everything of the intersection arithmetic that does not depend on the pixel ----------------
//   PLANE   g0 = z - eye_z
//   SPHERE  g0..2 = eye - centre, g3 = |eye - centre|^2 - r^2
//   CAPSULE g0..2 = ba = end1 - end0, g3..5 = oa = eye - end0, g6 = ba.ba, g7 = ba.oa, g8 = ba.ba oa.oa - (ba.oa)^2 - r^2 ba.ba,
//           g9 = oa.oa - r^2, g10 = |eye - end1|^2 - r^2                (a zero-length capsule is prepared as the SPHERE it is, and a
//           capsule the eye is inside of as a sphere no ray reaches)
//   CYL     g0, g1 = eye.xy - centre.xy, g2 = g0^2 + g1^2 - r^2, g3 = z0 - eye_z, g4 = z1 - eye_z, g5 = r^2
//   BOX     g0..2 = eye - centre in the box frame, g3..5 = half extents, g6 = cos, g7 = sin
//   OBOX    g0..2 = eye - centre in the box frame, g3..5 = half extents, g6..9 = the quaternion.  The ray is rotated into the box frame per
//           pixel (about 20 FMA) rather than kept as two prescaled axes plus a cross product: it fits g[11] with a word to spare, and the
//           slab test then reads the same words (eye in the box frame, half extents) as BOX's, so both share it.
// u0..v1: the screen-space bound the CUDA tile test reads (filled by the caller; the CPU checker does not cull).
struct SrlPrep { float type, g[11], u0, u1, v0, v1; };

SRL_RHD void srl_prepare(const float* eye, const SrlPrim& p, SrlPrep& q) {
    const int type = (int)p.type;
    q.type = p.type;
    for (int i = 0; i < 11; ++i) q.g[i] = 0.f;
    q.u0 = -1e30f; q.u1 = 1e30f; q.v0 = -1e30f; q.v1 = 1e30f;
    if (type == SRL_PRIM_PLANE) q.g[0] = p.a[0] - eye[2];
    else if (type == SRL_PRIM_SPHERE) {
        const float ox = eye[0] - p.a[0], oy = eye[1] - p.a[1], oz = eye[2] - p.a[2];
        q.g[0] = ox; q.g[1] = oy; q.g[2] = oz; q.g[3] = ox * ox + oy * oy + oz * oz - p.a[3] * p.a[3];
    } else if (type == SRL_PRIM_CAPSULE) {
        const float r = p.a[6];
        const float ba[3] = {p.a[3] - p.a[0], p.a[4] - p.a[1], p.a[5] - p.a[2]}, oa[3] = {eye[0] - p.a[0], eye[1] - p.a[1], eye[2] - p.a[2]};
        const float ob[3] = {eye[0] - p.a[3], eye[1] - p.a[4], eye[2] - p.a[5]};
        const float baba = ba[0] * ba[0] + ba[1] * ba[1] + ba[2] * ba[2], baoa = ba[0] * oa[0] + ba[1] * oa[1] + ba[2] * oa[2];
        const float oaoa = oa[0] * oa[0] + oa[1] * oa[1] + oa[2] * oa[2];
        const float k = baba < 1e-12f || baoa <= 0.f ? 0.f : baoa >= baba ? 1.f : baoa / baba;
        const float w[3] = {oa[0] - k * ba[0], oa[1] - k * ba[1], oa[2] - k * ba[2]};
        if (baba < 1e-12f || w[0] * w[0] + w[1] * w[1] + w[2] * w[2] < r * r) {
            // an eye inside the capsule sees no entry point (a solid seen from inside is not drawn, as for the other types; the end sphere
            // the ray leaves through is not its boundary there): prepared as a sphere no ray reaches
            q.type = (float)SRL_PRIM_SPHERE;
            q.g[0] = oa[0]; q.g[1] = oa[1]; q.g[2] = oa[2]; q.g[3] = baba < 1e-12f ? oaoa - r * r : 1e30f;
        } else {
            for (int i = 0; i < 3; ++i) { q.g[i] = ba[i]; q.g[3 + i] = oa[i]; }
            q.g[6] = baba; q.g[7] = baoa; q.g[8] = baba * oaoa - baoa * baoa - r * r * baba;
            q.g[9] = oaoa - r * r; q.g[10] = ob[0] * ob[0] + ob[1] * ob[1] + ob[2] * ob[2] - r * r;
        }
    } else if (type == SRL_PRIM_CYL) {
        const float ox = eye[0] - p.a[0], oy = eye[1] - p.a[1];
        q.g[0] = ox; q.g[1] = oy; q.g[2] = ox * ox + oy * oy - p.a[4] * p.a[4]; q.g[3] = p.a[2] - eye[2]; q.g[4] = p.a[3] - eye[2]; q.g[5] = p.a[4] * p.a[4];
    } else if (type == SRL_PRIM_OBOX) {
        const float o[3] = {eye[0] - p.a[0], eye[1] - p.a[1], eye[2] - p.a[2]};
        srl_quat_rotate_inv(p.a + 6, o, q.g);
        for (int i = 3; i < 10; ++i) q.g[i] = p.a[i];
    } else {
        const float cs = p.a[6], sn = p.a[7], px = eye[0] - p.a[0], py = eye[1] - p.a[1];
        q.g[0] = cs * px + sn * py; q.g[1] = -sn * px + cs * py; q.g[2] = eye[2] - p.a[2];
        q.g[3] = p.a[3]; q.g[4] = p.a[4]; q.g[5] = p.a[5]; q.g[6] = cs; q.g[7] = sn;
    }
}

// ---- ray (eye, unit d) against a prepared primitive: the nearest t > 1e-4, or false ----
SRL_RHD bool srl_sphere_t(float b, float cc, float& t) {          // b = (eye - c).d, cc = |eye - c|^2 - r^2
    const float h = b * b - cc;
    if (h < 0.f) return false;
    t = -b - sqrtf(h);
    return t > 1e-4f;
}
// OBOX = false compiles a caller that never sees an oriented box (the CUDA raster kernel for lists without distractor bodies) without its code
template <bool OBOX = true>
SRL_RHD bool srl_hit_t(const SrlPrep& q, const float* d, float& t) {
    const int type = (int)q.type;
    const float* g = q.g;
    if (type == SRL_PRIM_PLANE) {
        if (!(d[2] < -1e-6f)) return false;
        t = g[0] / d[2];
        return t > 1e-4f;
    }
    if (type == SRL_PRIM_SPHERE) return srl_sphere_t(g[0] * d[0] + g[1] * d[1] + g[2] * d[2], g[3], t);
    if (type == SRL_PRIM_CAPSULE) {
        // the segment end0-end1 swept by a sphere: the open cylinder between the ends first, else the nearer of the two end spheres
        const float bard = g[0] * d[0] + g[1] * d[1] + g[2] * d[2], rdoa = g[3] * d[0] + g[4] * d[1] + g[5] * d[2];
        const float a = g[6] - bard * bard, b = g[6] * rdoa - g[7] * bard;
        const float h = b * b - a * g[8];
        if (h >= 0.f && a > 1e-12f) {
            const float t0 = (-b - sqrtf(h)) / a;
            const float y = g[7] + t0 * bard;
            if (y > 0.f && y < g[6] && t0 > 1e-4f) { t = t0; return true; }
        }
        float t1 = 0.f, t2 = 0.f;
        const bool h1 = srl_sphere_t(rdoa, g[9], t1), h2 = srl_sphere_t(rdoa - bard, g[10], t2);
        if (h1 && (!h2 || t1 <= t2)) { t = t1; return true; }
        if (h2) { t = t2; return true; }
        return false;
    }
    if (type == SRL_PRIM_CYL) {
        float best = 1e30f;
        const float a = d[0] * d[0] + d[1] * d[1];
        if (a > 1e-12f) {                                  // side
            const float b = g[0] * d[0] + g[1] * d[1];
            const float h = b * b - a * g[2];
            if (h >= 0.f) {
                const float tt = (-b - sqrtf(h)) / a;
                const float z = tt * d[2];
                if (tt > 1e-4f && z >= g[3] && z <= g[4]) best = tt;
            }
        }
        if (fabsf(d[2]) > 1e-12f) {                        // the cap facing the ray
            const float tt = (d[2] < 0.f ? g[4] : g[3]) / d[2];
            const float x = g[0] + tt * d[0], y = g[1] + tt * d[1];
            if (tt > 1e-4f && tt < best && x * x + y * y <= g[5]) best = tt;
        }
        if (best > 1e29f) return false;
        t = best;
        return true;
    }
    // box: slabs in the box frame
    float ld[3];
    if (OBOX && type == SRL_PRIM_OBOX) srl_quat_rotate_inv(g + 6, d, ld);
    else { ld[0] = g[6] * d[0] + g[7] * d[1]; ld[1] = -g[7] * d[0] + g[6] * d[1]; ld[2] = d[2]; }
    float tn = -1e30f, tf = 1e30f;
    for (int k = 0; k < 3; ++k) {
        if (fabsf(ld[k]) < 1e-12f) { if (fabsf(g[k]) > g[3 + k]) return false; continue; }
        const float inv = 1.f / ld[k];
        float t0 = (-g[3 + k] - g[k]) * inv, t1 = (g[3 + k] - g[k]) * inv;
        if (t0 > t1) { const float tmp = t0; t0 = t1; t1 = tmp; }
        if (t0 > tn) tn = t0;
        if (t1 < tf) tf = t1;
    }
    if (tn > tf || tn <= 1e-4f) return false;
    t = tn;
    return true;
}

// the face of a box (half extents h) a point l in the box frame lies on: the axis whose slab it is closest to leaving, as a signed unit vector
SRL_RHD void srl_box_face(const float* l, const float* h, float* ln) {
    int axis = 0; float out = fabsf(l[0]) - h[0], la = l[0];          // la = l[axis], kept without indexing by a run-time axis (local memory)
    for (int k = 1; k < 3; ++k) { const float o = fabsf(l[k]) - h[k]; if (o > out) { out = o; axis = k; la = l[k]; } }
    const float sg = la < 0.f ? -1.f : 1.f;
    ln[0] = axis == 0 ? sg : 0.f; ln[1] = axis == 1 ? sg : 0.f; ln[2] = axis == 2 ? sg : 0.f;
}

// Outward unit normal of primitive p at the surface point P.
template <bool OBOX = true>
SRL_RHD void srl_normal_at(const SrlPrim& p, const float* P, float* n) {
    const int type = (int)p.type;
    n[0] = 0.f; n[1] = 0.f; n[2] = 1.f;
    if (type == SRL_PRIM_SPHERE) { for (int i = 0; i < 3; ++i) n[i] = (P[i] - p.a[i]) / p.a[3]; }
    else if (type == SRL_PRIM_CAPSULE) {
        const float ba[3] = {p.a[3] - p.a[0], p.a[4] - p.a[1], p.a[5] - p.a[2]}, w[3] = {P[0] - p.a[0], P[1] - p.a[1], P[2] - p.a[2]};
        const float baba = ba[0] * ba[0] + ba[1] * ba[1] + ba[2] * ba[2];
        float k = baba < 1e-12f ? 0.f : (w[0] * ba[0] + w[1] * ba[1] + w[2] * ba[2]) / baba;
        k = k < 0.f ? 0.f : k > 1.f ? 1.f : k;
        for (int i = 0; i < 3; ++i) n[i] = (w[i] - k * ba[i]) / p.a[6];
    } else if (type == SRL_PRIM_CYL) {
        const float rx = P[0] - p.a[0], ry = P[1] - p.a[1], r = p.a[4];
        if (rx * rx + ry * ry < 0.9999f * r * r) n[2] = P[2] > 0.5f * (p.a[2] + p.a[3]) ? 1.f : -1.f;      // on a cap
        else { n[0] = rx / r; n[1] = ry / r; n[2] = 0.f; }
    } else if (type == SRL_PRIM_BOX) {
        const float cs = p.a[6], sn = p.a[7], px = P[0] - p.a[0], py = P[1] - p.a[1];
        const float l[3] = {cs * px + sn * py, -sn * px + cs * py, P[2] - p.a[2]};
        float ln[3];
        srl_box_face(l, p.a + 3, ln);
        n[0] = cs * ln[0] - sn * ln[1]; n[1] = sn * ln[0] + cs * ln[1]; n[2] = ln[2];
    } else if (OBOX && type == SRL_PRIM_OBOX) {
        const float w[3] = {P[0] - p.a[0], P[1] - p.a[1], P[2] - p.a[2]};
        float l[3], ln[3];
        srl_quat_rotate_inv(p.a + 6, w, l);
        srl_box_face(l, p.a + 3, ln);
        srl_quat_rotate(p.a + 6, ln, n);
    }
}

// One pixel: nearest hit over the primitives whose bit is set in `mask` (in list order), ambient + Lambert shading, 8-bit RGB.  Row 0 is the
// TOP of the image (getCameraImage).  The CUDA kernel passes the subset whose screen bound reaches the pixel's neighbourhood; the CPU checker
// passes all of them.  `prep[k]` is srl_prepare(c.eye, prims[k]).
SRL_RHD unsigned long long srl_prim_mask_all(int np) { return np >= 64 ? ~0ull : ((1ull << np) - 1ull); }
template <bool OBOX = true>
SRL_RHD void srl_render_pixel(const SrlCam& c, const SrlPrep* prep, const SrlPrim* prims, unsigned long long mask, int x, int y, uint8_t* rgb) {
    const float u = c.ub + c.su * ((float)x + 0.5f);
    const float v = c.vb - c.sv * ((float)y + 0.5f);
    float d[3] = {c.fwd[0] + u * c.right[0] + v * c.up[0], c.fwd[1] + u * c.right[1] + v * c.up[1], c.fwd[2] + u * c.right[2] + v * c.up[2]};
    const float dl = 1.f / sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    d[0] *= dl; d[1] *= dl; d[2] *= dl;
    float best = 1e30f;
    int win = -1;
    while (mask) {
#if defined(__CUDA_ARCH__)
        const int k = __ffsll((long long)mask) - 1;
#else
        const int k = __builtin_ctzll(mask);
#endif
        mask &= mask - 1ull;
        float t = 0.f;
        if (srl_hit_t<OBOX>(prep[k], d, t) && t < best) { best = t; win = k; }
    }
    float shade = 1.f, col[3] = {0.84f, 0.89f, 0.95f};                 // background (above the horizon)
    if (win >= 0) {
        const SrlPrim& p = prims[win];
        const float P[3] = {c.eye[0] + best * d[0], c.eye[1] + best * d[1], c.eye[2] + best * d[2]};
        float n[3];
        srl_normal_at<OBOX>(p, P, n);
        col[0] = p.r; col[1] = p.g; col[2] = p.b;
        if ((int)p.type == SRL_PRIM_PLANE && p.a[1] > 0.f) {
            const int ix = (int)floorf(P[0] / p.a[1]), iy = (int)floorf(P[1] / p.a[1]);
            if ((ix + iy) & 1) { col[0] = p.a[2]; col[1] = p.a[3]; col[2] = p.a[4]; }
        }
        const float L[3] = {0.3713907f, 0.5570860f, 0.7427814f};     // normalised (2, 3, 4): one fixed directional light, no shadows
        const float nl = n[0] * L[0] + n[1] * L[1] + n[2] * L[2];
        shade = 0.55f + 0.45f * (nl > 0.f ? nl : 0.f);
    }
    for (int k = 0; k < 3; ++k) {
        float vv = col[k] * shade * 255.f + 0.5f;
        vv = vv < 0.f ? 0.f : vv > 255.f ? 255.f : vv;
        rgb[k] = (uint8_t)vv;
    }
}

// ---- scene builders (shared so that both implementations draw the same list) ------------------------------------------------------
struct SrlKukaSceneConst {      // from the model blob / KukaParams
    float base[3];
    float table_z, txmin, txmax, tymin, tymax;
    float glider_z, disc_r, disc_z0, disc_z1, stack_r, stack_top;
    int two_buttons;
};

// joint_p: world origins of the 12 movable joint frames (bodies 0..7 chain, 8-9 finger A, 10-11 finger B); sph: world centres + radii of the
// collision spheres of the gripper bodies (body >= 7).  Returns the number of primitives written (<= SRL_MAX_PRIMS).
SRL_RHD int srl_kuka_scene(const SrlKukaSceneConst& K, const float* joint_p, const float* sph, int nsph, float bbx, float bby, float bbz, float qb,
                           float bb2x, float bb2y, float b2z, float qb2, SrlPrim* out) {
    int n = 0;
    srl_prim_plane(out[n++], -1.0f, 1.0f, 1.0f, 1.0f, 1.0f);                                            // plane.urdf at z = -1 (kuka_button_gym_env.py:222)
    const float tcx = 0.5f * (K.txmin + K.txmax), tcy = 0.5f * (K.tymin + K.tymax), thx = 0.5f * (K.txmax - K.txmin), thy = 0.5f * (K.tymax - K.tymin);
    srl_prim_box(out[n++], tcx, tcy, K.table_z - 0.025f, thx, thy, 0.025f, 1.f, 0.f, 0.92f, 0.82f, 0.68f);   // table top slab (5 cm), light wood
    for (int k = 0; k < 4; ++k)                                                                           // legs down to the plane
        srl_prim_box(out[n++], tcx + ((k & 1) ? 1.f : -1.f) * (thx - 0.1f), tcy + ((k & 2) ? 1.f : -1.f) * (thy - 0.1f), 0.5f * (K.table_z - 0.05f - 1.0f),
                     0.05f, 0.05f, 0.5f * (K.table_z - 0.05f + 1.0f), 1.f, 0.f, 0.85f, 0.75f, 0.62f);
    // button(s): base + fixed cylinder stack (green), pressable disc (yellow) -- colours of urdf/simple_button.urdf
    for (int b = 0; b < (K.two_buttons ? 2 : 1); ++b) {
        const float x = b ? bb2x : bbx, y = b ? bb2y : bby, z = b ? b2z : bbz, q = b ? qb2 : qb;
        srl_prim_cyl(out[n++], x, y, z, z + K.stack_top, K.stack_r, 0.f, 1.f, 0.f);
        srl_prim_cyl(out[n++], x, y, z + K.glider_z + q + K.disc_z0, z + K.glider_z + q + K.disc_z1, K.disc_r, 1.f, 1.f, 0.f);
    }
    // arm: fixed pedestal, then a capsule per link between consecutive joint frames (iiwa orange / grey, RECALLED materials)
    srl_prim_capsule(out[n++], K.base, joint_p, 0.075f, 0.30f, 0.30f, 0.30f);
    for (int i = 0; i < 7; ++i) {
        const bool orange = (i & 1) == 0;          // orange links alternating with blue-grey ones, as in imgs/kuka.gif
        srl_prim_capsule(out[n++], joint_p + 3 * i, joint_p + 3 * (i + 1), i < 4 ? 0.065f : 0.055f, orange ? 1.0f : 0.5f, orange ? 0.42f : 0.7f, orange ? 0.04f : 1.0f);
    }
    // gripper: base to the two fingers, finger links, plus the collision spheres of the gripper bodies
    srl_prim_capsule(out[n++], joint_p + 21, joint_p + 24, 0.02f, 0.15f, 0.15f, 0.15f);
    srl_prim_capsule(out[n++], joint_p + 24, joint_p + 27, 0.012f, 0.15f, 0.15f, 0.15f);
    srl_prim_capsule(out[n++], joint_p + 21, joint_p + 30, 0.02f, 0.15f, 0.15f, 0.15f);
    srl_prim_capsule(out[n++], joint_p + 30, joint_p + 33, 0.012f, 0.15f, 0.15f, 0.15f);
    for (int k = 0; k < nsph && n < SRL_MAX_PRIMS; ++k) srl_prim_sphere(out[n++], sph + 4 * k, sph[4 * k + 3], 0.2f, 0.2f, 0.2f);
    return n;
}

// KukaRandButton's distractor bodies: per object type the drawing words of the asset blob (distractor_core.h DC_A_SHAPE / DC_A_HALF /
// DC_A_RGB; srl_sim/model.py: distractor_blob), checked by dc_blob_error.
struct SrlBodyLooks { float shape[DC_NTYPE], half[DC_NTYPE][3], rgb[DC_NTYPE][3]; };
SRL_RHD void srl_body_looks(const double* blob, SrlBodyLooks& L) {
    for (int t = 0; t < DC_NTYPE; ++t) {
        const double* w = blob + t * DC_TYPE_WORDS;
        L.shape[t] = (float)w[DC_A_SHAPE];
        for (int i = 0; i < 3; ++i) { L.half[t][i] = (float)w[DC_A_HALF + i]; L.rgb[t][i] = (float)w[DC_A_RGB + i]; }
    }
}

// The present bodies of one env (B: DC_NBODY x DC_B_WORDS, distractor_core.h) appended to a scene list of n primitives: shape 0 a box of the
// type's half extents at the body's pose, shape 1 a sphere of radius half[0].  They come after the scene, and the nearest-hit search takes
// a later primitive only when it is strictly nearer, so the pixels no body covers keep the bytes they have without bodies.
SRL_RHD int srl_distractor_prims(const SrlBodyLooks& L, const float* B, int n, SrlPrim* out) {
    for (int k = 0; k < DC_NBODY && n < SRL_MAX_PRIMS; ++k) {
        const float* b = B + k * DC_B_WORDS;
        if (b[DC_B_PRESENT] == 0.f) continue;
        const int t = (int)b[DC_B_TYPE];
        if (L.shape[t] == 1.f) srl_prim_sphere(out[n++], b + DC_B_P, L.half[t][0], L.rgb[t][0], L.rgb[t][1], L.rgb[t][2]);
        else srl_prim_obox(out[n++], b + DC_B_P, L.half[t], b + DC_B_Q, L.rgb[t][0], L.rgb[t][1], L.rgb[t][2]);
    }
    return n;
}

// MobileRobot family: plane, four walls (urdf/wall.urdf: box 4 x 0.1 x 0.1; left red, bottom black, right green, top blue:
// mobile_robot_env.py:184-203), the robot as a box of the racecar's footprint, the target(s).
// kind: 0 base, 3 one-dimensional, 1 two targets, 2 line target (urdf/wall_target.urdf: box 4 x 0.5 x 0.1, yellow, rotated by pi / 2).
SRL_RHD int srl_mobile_scene(int kind, float rx, float ry, float t0x, float t0y, float t1x, float t1y, SrlPrim* out) {
    int n = 0;
    srl_prim_plane(out[n++], 0.f, 1.0f, 1.0f, 1.0f, 1.0f);
    srl_prim_box(out[n++], 2.f, 0.f, 0.f, 2.f, 0.05f, 0.05f, 1.f, 0.f, 0.8f, 0.f, 0.f);
    if (kind != 3) {            // the 1-D variant only has the left wall (mobile_robot_1D_env.py:84-86)
        srl_prim_box(out[n++], 4.f, 2.f, 0.f, 2.f, 0.05f, 0.05f, 0.f, 1.f, 0.f, 0.f, 0.f);
        srl_prim_box(out[n++], 2.f, 4.f, 0.f, 2.f, 0.05f, 0.05f, 1.f, 0.f, 0.f, 0.8f, 0.f);
        srl_prim_box(out[n++], 0.f, 2.f, 0.f, 2.f, 0.05f, 0.05f, 0.f, 1.f, 0.f, 0.f, 0.8f);
    }
    if (kind == 2) srl_prim_box(out[n++], t0x, 2.f, -0.045f, 2.f, 0.25f, 0.05f, 0.f, 1.f, 1.f, 1.f, 0.f);
    else {
        srl_prim_cyl(out[n++], t0x, t0y, 0.f, 0.03f, 0.18f, 1.f, 1.f, 0.f);                                // urdf/cylinder.urdf: the button disc mesh (r 0.09) scaled (2, 2, 1), yellow
        if (kind == 1) srl_prim_cyl(out[n++], t1x, t1y, 0.f, 0.03f, 0.18f, 0.8f, 0.f, 0.f);                 // second target recoloured red (mobile_robot_2target_env.py:71)
    }
    srl_prim_box(out[n++], rx, ry, 0.09f, 0.325f, 0.1f, 0.07f, 1.f, 0.f, 0.1f, 0.2f, 0.8f);                // racecar footprint ROBOT_LENGTH x ROBOT_WIDTH (:27-28), blue as in imgs/mobile_robot.gif
    srl_prim_box(out[n++], rx + 0.1f, ry, 0.17f, 0.12f, 0.08f, 0.03f, 1.f, 0.f, 0.95f, 0.95f, 0.95f);      // a white cabin so that the heading side is visible
    return n;
}
