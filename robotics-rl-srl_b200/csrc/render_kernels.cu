// Image observations for the batched simulator (SURVEY.md 8(f).4): one launch builds every env's primitive list from its state, one launch
// ray-casts all frames.  Per-pixel arithmetic and the scene lists live in render_core.h (shared with the CPU checker).
//
// Layout: the primitive lists are [N][SRL_MAX_PRIMS][16 floats] in HBM (3 KB per env), and so are their per-camera prepared forms (the
// pixel-independent part of the intersection arithmetic + a screen-space bound).  The raster kernel runs one CTA of 32 x 16 pixels per
// (tile, env): it stages the env's prepared list in shared memory once, each warp keeps the primitives whose bound reaches its 8 x 8 pixel
// block, and the RGB bytes go out row-major -- a 224 x 224 frame is 98 tiles, 4096 envs are 401 k CTAs, 617 MB of output per call.
#include "common.cuh"
#include "render_core.h"

namespace {

__global__ void mobile_prims_kernel(MobileDev d, int n, int kind, float* __restrict__ prims, int* __restrict__ counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double2 pos = d.pos[i], t0 = d.tgt0[i], t1 = d.tgt1[i];
    const int rk = kind == SRL_ENV_MOBILE_2TARGET ? 1 : kind == SRL_ENV_MOBILE_LINE_TARGET ? 2 : kind == SRL_ENV_MOBILE_1D ? 3 : 0;
    SrlPrim* out = reinterpret_cast<SrlPrim*>(prims + (size_t)i * SRL_MAX_PRIMS * SRL_PRIM_WORDS);
    counts[i] = srl_mobile_scene(rk, (float)pos.x, (float)pos.y, (float)t0.x, (float)t0.y, (float)t1.x, (float)t1.y, out);
}

// Screen-space bound of a primitive: [u0, u1] x [v0, v1] in the units of the pixel rays (direction = fwd + u right + v up), covering every
// ray that can touch it.  false = "cannot bound" (the plane, or a primitive that reaches behind the eye plane): such a primitive is always kept.
struct ScreenRect { float u0, u1, v0, v1; };

__device__ __forceinline__ void cam_space(const SrlCam& c, float x, float y, float z, float* o) {
    const float px = x - c.eye[0], py = y - c.eye[1], pz = z - c.eye[2];
    o[0] = px * c.right[0] + py * c.right[1] + pz * c.right[2];
    o[1] = px * c.up[0] + py * c.up[1] + pz * c.up[2];
    o[2] = px * c.fwd[0] + py * c.fwd[1] + pz * c.fwd[2];
}
__device__ __forceinline__ bool rect_point(ScreenRect& r, const float* q) {
    if (q[2] < 1e-3f) return false;
    const float iz = 1.f / q[2], u = q[0] * iz, v = q[1] * iz;
    r.u0 = fminf(r.u0, u); r.u1 = fmaxf(r.u1, u); r.v0 = fminf(r.v0, v); r.v1 = fmaxf(r.v1, v);
    return true;
}
// sphere: per axis the two tangent directions from the eye of the circle (x, z), radius R -- slopes (x z -+ R sqrt(x^2 + z^2 - R^2)) / (z^2 - R^2)
__device__ __forceinline__ bool rect_sphere(ScreenRect& r, const float* q, float R) {
    R = R * 1.001f + 1e-4f;
    if (q[2] < R * 1.01f + 1e-3f) return false;
    const float den = 1.f / (q[2] * q[2] - R * R);
    const float su = R * sqrtf(fmaxf(q[0] * q[0] + q[2] * q[2] - R * R, 0.f)), sv = R * sqrtf(fmaxf(q[1] * q[1] + q[2] * q[2] - R * R, 0.f));
    r.u0 = fminf(r.u0, (q[0] * q[2] - su) * den); r.u1 = fmaxf(r.u1, (q[0] * q[2] + su) * den);
    r.v0 = fminf(r.v0, (q[1] * q[2] - sv) * den); r.v1 = fmaxf(r.v1, (q[1] * q[2] + sv) * den);
    return true;
}
__device__ __forceinline__ bool prim_rect(const SrlCam& c, const SrlPrim& p, ScreenRect& r) {
    const int type = (int)p.type;
    r.u0 = 1e30f; r.u1 = -1e30f; r.v0 = 1e30f; r.v1 = -1e30f;
    float q[3];
    if (type == SRL_PRIM_SPHERE) { cam_space(c, p.a[0], p.a[1], p.a[2], q); return rect_sphere(r, q, p.a[3]); }
    if (type == SRL_PRIM_CAPSULE) {                       // convex hull of the two end spheres: the union of their bounds bounds it
        cam_space(c, p.a[0], p.a[1], p.a[2], q);
        if (!rect_sphere(r, q, p.a[6])) return false;
        cam_space(c, p.a[3], p.a[4], p.a[5], q);
        return rect_sphere(r, q, p.a[6]);
    }
    if (type == SRL_PRIM_CYL || type == SRL_PRIM_BOX) {   // the 8 corners of the box (of the cylinder's bounding box)
        const bool cyl = type == SRL_PRIM_CYL;
        const float cx = p.a[0], cy = p.a[1], cz = cyl ? 0.5f * (p.a[2] + p.a[3]) : p.a[2];
        const float hx = (cyl ? p.a[4] : p.a[3]) * 1.001f + 1e-4f, hy = (cyl ? p.a[4] : p.a[4]) * 1.001f + 1e-4f, hz = (cyl ? 0.5f * (p.a[3] - p.a[2]) : p.a[5]) * 1.001f + 1e-4f;
        const float cs = cyl ? 1.f : p.a[6], sn = cyl ? 0.f : p.a[7];
        bool ok = true;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float lx = (k & 1) ? hx : -hx, ly = (k & 2) ? hy : -hy, lz = (k & 4) ? hz : -hz;
            cam_space(c, cx + cs * lx - sn * ly, cy + sn * lx + cs * ly, cz + lz, q);
            ok = rect_point(r, q) && ok;
        }
        return ok;
    }
    if (type == SRL_PRIM_OBOX) {                          // its 8 rotated corners, padded as BOX's
        bool ok = true;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float l[3] = {((k & 1) ? 1.f : -1.f) * (p.a[3] * 1.001f + 1e-4f), ((k & 2) ? 1.f : -1.f) * (p.a[4] * 1.001f + 1e-4f),
                                ((k & 4) ? 1.f : -1.f) * (p.a[5] * 1.001f + 1e-4f)};
            float w[3];
            srl_quat_rotate(p.a + 6, l, w);
            cam_space(c, p.a[0] + w[0], p.a[1] + w[1], p.a[2] + w[2], q);
            ok = rect_point(r, q) && ok;
        }
        return ok;
    }
    return false;
}

// One thread per (env, primitive): the per-camera prepared form (render_core.h) plus the screen-space bound, [N][SRL_MAX_PRIMS][16 floats].
__global__ void prepare_kernel(const float* __restrict__ prims, const int* __restrict__ counts, SrlCam cam, int n, float* __restrict__ prep) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int env = i / SRL_MAX_PRIMS, k = i % SRL_MAX_PRIMS;
    if (env >= n || k >= counts[env]) return;
    const SrlPrim p = reinterpret_cast<const SrlPrim*>(prims)[i];
    SrlPrep q;
    srl_prepare(cam.eye, p, q);
    ScreenRect r;
    if (prim_rect(cam, p, r)) { q.u0 = r.u0; q.u1 = r.u1; q.v0 = r.v0; q.v1 = r.v1; }       // else: srl_prepare's "everywhere"
    reinterpret_cast<SrlPrep*>(prep)[i] = q;
}
// the same with one camera per env (srl_sim_render_cameras): the thread takes cams[env]
__global__ void prepare_cams_kernel(const float* __restrict__ prims, const int* __restrict__ counts, const SrlCam* __restrict__ cams, int n,
                                    float* __restrict__ prep) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int env = i / SRL_MAX_PRIMS, k = i % SRL_MAX_PRIMS;
    if (env >= n || k >= counts[env]) return;
    const SrlCam cam = cams[env];
    const SrlPrim p = reinterpret_cast<const SrlPrim*>(prims)[i];
    SrlPrep q;
    srl_prepare(cam.eye, p, q);
    ScreenRect r;
    if (prim_rect(cam, p, r)) { q.u0 = r.u0; q.u1 = r.u1; q.v0 = r.v0; q.v1 = r.v1; }
    reinterpret_cast<SrlPrep*>(prep)[i] = q;
}

// follow_robot: one thread per env finishes its camera from the robot's position, as the host would for the target
// float32(float64 position + float64 offset) (srl_camera_target gives the host's bits)
__global__ void follow_cams_kernel(const SrlCamFollow* __restrict__ in, const double2* __restrict__ pos, int n, SrlCam* __restrict__ cams) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const SrlCamFollow f = in[i];
    const double2 p = pos[i];
    const float target[3] = {(float)(p.x + (double)f.off[0]), (float)(p.y + (double)f.off[1]), f.off[2]};
    SrlCam c;
    srl_camera_target(target, f.a, c);
    cams[i] = c;
}

// One CTA = one 32 x 16 pixel tile of one env's frame, one warp = an 8 x 8 pixel block of it (two pixels per thread, four rows apart).  Each
// warp first tests, one lane per primitive, whether the primitive's screen-space bound overlaps its block (conservative: a dropped primitive
// cannot be hit by any pixel of the block, so the nearest-hit search over the kept ones -- in list order -- returns what the search over the
// full list does); its pixels then ray-cast the kept ones, and the tile's RGB bytes go out as 32-bit words (96 contiguous bytes per tile row)
// when the frame geometry allows.  grid = (tiles across, tiles down, envs).
#define SRL_TILE_W 32
#define SRL_TILE_H 16
// BODIES: the lists may hold oriented boxes (a Kuka handle with distractor bodies); the kernel for the other lists leaves their code out.
// The body is shared by raster_kernel (one camera, a kernel parameter) and raster_cams_kernel (one camera per env, staged in shared memory
// before the __syncthreads below).
template <bool CULL, bool BODIES>
__device__ __forceinline__ void raster_tile(const float* __restrict__ prims, const float* __restrict__ prep, const int* __restrict__ counts, const SrlCam& cam,
                                            int W, int H, uint8_t* __restrict__ rgb) {
    static_assert(SRL_MAX_PRIMS <= 64, "the kept set is a 64-bit mask");
    __shared__ __align__(16) SrlPrep sq[SRL_MAX_PRIMS];
    __shared__ __align__(16) uint8_t tile[SRL_TILE_H][3 * SRL_TILE_W];
    const int env = blockIdx.z;
    const int np = counts[env];
    const float4* src = reinterpret_cast<const float4*>(prep + (size_t)env * SRL_MAX_PRIMS * SRL_PRIM_WORDS);
    for (int k = threadIdx.x; k < np * (SRL_PRIM_WORDS / 4); k += blockDim.x) reinterpret_cast<float4*>(sq)[k] = src[k];
    __syncthreads();
    const int x0 = blockIdx.x * SRL_TILE_W, y0 = blockIdx.y * SRL_TILE_H;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bx = (warp & 3) * 8, by = (warp >> 2) * 8;               // this warp's block inside the tile
    unsigned long long mask = srl_prim_mask_all(np);
    if (CULL) {
        const float xa = (float)(x0 + bx), ya = (float)(y0 + by), xb = (float)min(x0 + bx + 8, W), yb = (float)min(y0 + by + 8, H);   // pixel EDGES
        const float tu0 = cam.ub + cam.su * xa, tu1 = cam.ub + cam.su * xb, tv1 = cam.vb - cam.sv * ya, tv0 = cam.vb - cam.sv * yb;
        const float eu = 1e-4f * (1.f + fmaxf(fabsf(tu0), fabsf(tu1))), ev = 1e-4f * (1.f + fmaxf(fabsf(tv0), fabsf(tv1)));
        unsigned w[2];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int k = lane + 32 * half;
            bool keep = k < np;
            if (keep) {
                const SrlPrep& q = sq[k];
                keep = q.u1 >= tu0 - eu && q.u0 <= tu1 + eu && q.v1 >= tv0 - ev && q.v0 <= tv1 + ev;
            }
            w[half] = __ballot_sync(0xffffffffu, keep);
        }
        mask = (unsigned long long)w[0] | ((unsigned long long)w[1] << 32);
    }
    const SrlPrim* mine = reinterpret_cast<const SrlPrim*>(prims) + (size_t)env * SRL_MAX_PRIMS;
    const int lx = bx + (lane & 7), x = x0 + lx;
    const bool words = (W % SRL_TILE_W) == 0 && (H % SRL_TILE_H) == 0;   // whole tiles and 4-byte aligned rows (3 W is then a multiple of 96)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int ly = by + (lane >> 3) + 4 * r, y = y0 + ly;
        if (x < W && y < H) {
            uint8_t px[3];
            srl_render_pixel<BODIES>(cam, sq, mine, mask, x, y, px);
            if (words) { tile[ly][3 * lx] = px[0]; tile[ly][3 * lx + 1] = px[1]; tile[ly][3 * lx + 2] = px[2]; }
            else {
                uint8_t* o = rgb + ((size_t)env * H * W + (size_t)y * W + x) * 3;
                o[0] = px[0]; o[1] = px[1]; o[2] = px[2];
            }
        }
    }
    if (!words) return;
    __syncthreads();
    for (int i = threadIdx.x; i < SRL_TILE_H * 24; i += blockDim.x) {
        const int row = i / 24, w = i % 24;
        uint32_t* o = reinterpret_cast<uint32_t*>(rgb + ((size_t)env * H * W + (size_t)(y0 + row) * W + x0) * 3);
        o[w] = reinterpret_cast<const uint32_t*>(tile[row])[w];
    }
}
template <bool CULL, bool BODIES>
__global__ void __launch_bounds__(256) raster_kernel(const float* __restrict__ prims, const float* __restrict__ prep, const int* __restrict__ counts, SrlCam cam,
                                                      int W, int H, uint8_t* __restrict__ rgb) {
    raster_tile<CULL, BODIES>(prims, prep, counts, cam, W, H, rgb);
}
// one camera per env: the CTA loads cams[env] (64 bytes) into shared memory once, for the culling test and the pixel rays
template <bool CULL, bool BODIES>
__global__ void __launch_bounds__(256) raster_cams_kernel(const float* __restrict__ prims, const float* __restrict__ prep, const int* __restrict__ counts,
                                                           const SrlCam* __restrict__ cams, int W, int H, uint8_t* __restrict__ rgb) {
    static_assert(sizeof(SrlCam) % 16 == 0, "the camera is staged as float4 words");
    __shared__ __align__(16) SrlCam scam;
    if (threadIdx.x < sizeof(SrlCam) / 16) reinterpret_cast<float4*>(&scam)[threadIdx.x] = reinterpret_cast<const float4*>(cams + blockIdx.z)[threadIdx.x];
    raster_tile<CULL, BODIES>(prims, prep, counts, scam, W, H, rgb);
}

// every env's frame from the prepared lists: through one camera (cam) or through cams[env] (cams != nullptr, device memory)
template <bool CULL, bool BODIES>
void raster_launch(dim3 grid, const float* pr, const float* pp, const int* cn, const SrlCam& cam, const SrlCam* cams, int W, int H, uint8_t* out, cudaStream_t st) {
    if (cams) raster_cams_kernel<CULL, BODIES><<<grid, 256, 0, st>>>(pr, pp, cn, cams, W, H, out);
    else raster_kernel<CULL, BODIES><<<grid, 256, 0, st>>>(pr, pp, cn, cam, W, H, out);
}
int raster_frames(srl_sim* s, const SrlCam& cam, const SrlCam* cams, int width, int height, uint8_t* rgb, cudaStream_t st) {
    const bool no_cull = getenv("SRL_RENDER_NO_CULL") != nullptr;       // debugging aid: the block test is conservative, so both paths give the same bytes (tests/test_render_gpu.py)
    const size_t per_env = (size_t)SRL_MAX_PRIMS * SRL_PRIM_WORDS;
    const bool bodies = s->dist != nullptr;
    for (int e0 = 0; e0 < s->n; e0 += 65535) {                           // grid.z is limited to 65535
        const dim3 grid((width + SRL_TILE_W - 1) / SRL_TILE_W, (height + SRL_TILE_H - 1) / SRL_TILE_H, min(65535, s->n - e0));
        uint8_t* out = rgb + (size_t)e0 * height * width * 3;
        const float* pr = s->render_prims + e0 * per_env; const float* pp = s->render_prep + e0 * per_env; const int* cn = s->render_counts + e0;
        const SrlCam* cm = cams ? cams + e0 : nullptr;
        if (bodies) {
            if (no_cull) raster_launch<false, true>(grid, pr, pp, cn, cam, cm, width, height, out, st);
            else raster_launch<true, true>(grid, pr, pp, cn, cam, cm, width, height, out, st);
        } else {
            if (no_cull) raster_launch<false, false>(grid, pr, pp, cn, cam, cm, width, height, out, st);
            else raster_launch<true, false>(grid, pr, pp, cn, cam, cm, width, height, out, st);
        }
    }
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

// every env's primitive list from its state, into the buffers allocated on first use
int render_lists(srl_sim* s, cudaStream_t st) {
    if (!s->render_prims) {
        SRL_CUDA_OK(cudaMalloc(&s->render_prims, (size_t)s->n * SRL_MAX_PRIMS * SRL_PRIM_WORDS * sizeof(float)));
        SRL_CUDA_OK(cudaMalloc(&s->render_prep, (size_t)s->n * SRL_MAX_PRIMS * SRL_PRIM_WORDS * sizeof(float)));
        SRL_CUDA_OK(cudaMalloc(&s->render_counts, (size_t)s->n * sizeof(int)));
    }
    if (srl_is_mobile(s->kind)) {
        mobile_prims_kernel<<<(s->n + 127) / 128, 128, 0, st>>>(s->mob, s->n, s->kind, s->render_prims, s->render_counts);
        SRL_CUDA_OK(cudaGetLastError());
        return 0;
    }
    return kuka_render_prims(s, s->render_prims, s->render_counts, st);
}

}  // namespace

int render_launch(srl_sim* s, const srl_camera* cam, int width, int height, uint8_t* rgb, cudaStream_t st) {
    if (render_lists(s, st)) return 1;
    SrlCam c;
    srl_camera_setup(cam->target, cam->distance, cam->yaw, cam->pitch, cam->roll, cam->fov, width, height, c);
    prepare_kernel<<<(s->n * SRL_MAX_PRIMS + 255) / 256, 256, 0, st>>>(s->render_prims, s->render_counts, c, s->n, s->render_prep);
    if (raster_frames(s, c, nullptr, width, height, rgb, st)) return 1;
    s->launches += 3;
    return 0;
}

// One camera per env.  The host builds the cameras (every env's SrlCam, or with follow_robot its angle part and target offset) into a pinned
// staging buffer and uploads them on the stream; the handle keeps the last camera array it built (with the size and follow_robot) and skips
// both when a call passes the same bytes again, so a loop that renders through the same cameras every step does no host work per call.
int render_cams_launch(srl_sim* s, const srl_camera* cams, int follow_robot, int width, int height, uint8_t* rgb, cudaStream_t st) {
    if (render_lists(s, st)) return 1;
    const size_t n = (size_t)s->n;
    if (!s->render_cam_key) {       // allocated last: a call after a failed allocation retries the missing buffers
        if (!s->render_cams) SRL_CUDA_OK(cudaMalloc(&s->render_cams, n * sizeof(SrlCam)));
        if (!s->render_follow) SRL_CUDA_OK(cudaMalloc(&s->render_follow, n * sizeof(SrlCamFollow)));
        if (!s->render_cam_stage)
            SRL_CUDA_OK(cudaMallocHost(&s->render_cam_stage, n * (sizeof(SrlCamFollow) > sizeof(SrlCam) ? sizeof(SrlCamFollow) : sizeof(SrlCam))));
        if (!s->render_cam_ev) SRL_CUDA_OK(cudaEventCreateWithFlags(&s->render_cam_ev, cudaEventDisableTiming));
        s->render_cam_key = (srl_camera*)malloc(n * sizeof(srl_camera));
        if (!s->render_cam_key) { srl_set_error("render_cameras: out of memory"); return 1; }
        s->render_cam_valid = 0;
    }
    const bool same = s->render_cam_valid && s->render_cam_follow == follow_robot && s->render_cam_w == width && s->render_cam_h == height &&
                      memcmp(s->render_cam_key, cams, n * sizeof(srl_camera)) == 0;
    if (!same) {
        s->render_cam_valid = 0;
        SRL_CUDA_OK(cudaEventSynchronize(s->render_cam_ev));            // the previous upload has left the staging buffer
        if (follow_robot) {
            SrlCamFollow* f = reinterpret_cast<SrlCamFollow*>(s->render_cam_stage);
            for (size_t i = 0; i < n; ++i) {
                const srl_camera& c = cams[i];
                srl_camera_angles(c.distance, c.yaw, c.pitch, c.roll, c.fov, width, height, f[i].a);
                for (int k = 0; k < 3; ++k) f[i].off[k] = c.target[k];
            }
            SRL_CUDA_OK(cudaMemcpyAsync(s->render_follow, f, n * sizeof(SrlCamFollow), cudaMemcpyHostToDevice, st));
        } else {
            SrlCam* o = reinterpret_cast<SrlCam*>(s->render_cam_stage);
            for (size_t i = 0; i < n; ++i) {
                const srl_camera& c = cams[i];
                srl_camera_setup(c.target, c.distance, c.yaw, c.pitch, c.roll, c.fov, width, height, o[i]);
            }
            SRL_CUDA_OK(cudaMemcpyAsync(s->render_cams, o, n * sizeof(SrlCam), cudaMemcpyHostToDevice, st));
        }
        SRL_CUDA_OK(cudaEventRecord(s->render_cam_ev, st));
        memcpy(s->render_cam_key, cams, n * sizeof(srl_camera));
        s->render_cam_follow = follow_robot; s->render_cam_w = width; s->render_cam_h = height;
        s->render_cam_valid = 1;
    }
    if (follow_robot) {     // the targets move with the robots: finish every camera from the current positions, on the device
        follow_cams_kernel<<<(s->n + 127) / 128, 128, 0, st>>>(s->render_follow, s->mob.pos, s->n, s->render_cams);
        s->launches += 1;
    }
    prepare_cams_kernel<<<(s->n * SRL_MAX_PRIMS + 255) / 256, 256, 0, st>>>(s->render_prims, s->render_counts, s->render_cams, s->n, s->render_prep);
    if (raster_frames(s, SrlCam{}, s->render_cams, width, height, rgb, st)) return 1;
    s->launches += 3;
    return 0;
}

void render_free(srl_sim* s) {
    if (s->render_prims) cudaFree(s->render_prims);
    if (s->render_prep) cudaFree(s->render_prep);
    if (s->render_counts) cudaFree(s->render_counts);
    if (s->render_cams) cudaFree(s->render_cams);
    if (s->render_follow) cudaFree(s->render_follow);
    if (s->render_cam_stage) cudaFreeHost(s->render_cam_stage);
    if (s->render_cam_ev) cudaEventDestroy(s->render_cam_ev);
    free(s->render_cam_key);
    s->render_prims = nullptr; s->render_prep = nullptr; s->render_counts = nullptr;
    s->render_cams = nullptr; s->render_follow = nullptr; s->render_cam_stage = nullptr; s->render_cam_ev = nullptr; s->render_cam_key = nullptr;
    s->render_cam_valid = 0;
}
