// Kuka state and trace format shared by the arm's kernels (kuka_kernels.cu) and the distractor bodies (distractor_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include "kuka_params.cuh"

// Per-env state in HBM, one 16-byte record per array: the live state (KukaDev) and the next-episode records (KukaNext) alike.
struct KukaState {
    float4* q[3];    // [N] joint positions  (12 floats as 3 x float4)
    float4* qd[3];   // [N] joint velocities
    float4* misc0;   // ee.x ee.y ee.z qb
    float4* misc1;   // qdb btn_base.x btn_base.y ep_ret
    float4* tgt;     // button_pos.xyz, button base z
    float4* grip;    // gripper_pos.xyz, signed button speed
    float4* eepos;   // link-6 origin xyz, moving button: low word of the float64 target y
    int4*   cnt;     // counter, n_contacts, n_outside, terminated | cbutton << 1 | ctable << 2
    int4*   cnt2;    // episode, total_steps, ep_len, moving button: high word of the float64 target y / two buttons: n_contacts[1]
    float4* btn2;    // two buttons only: second glider q, qd, second button base x, y
};

struct KukaDev : KukaState {
    KukaParams P;
    int epw;         // live env slots per warp (lanes, or groups of 4 lanes when coop)
    int coop;        // 1: four lanes per env (kuka_coop.cuh), epw <= 8
};

// The trace a traced kuka_kernel launch writes and distractor_kernel replays: per env and micro-step, the configuration the micro-step starts
// from and its kind as float4 records trace[(micro-step * 4 + r) * N + env]: q[0-3], q[4-7], q[8-11], (glider q, button base x y, tag | episode << 4).
// Tags: inside reset(), first micro-step of a reset() (the bodies are placed and settled before it), host-supplied placements, the kick.
enum { DT_RESET = 1, DT_FIRST = 2, DT_HOST_DRAWS = 4, DT_KICK = 8 };
// reset_draws row width with distractor bodies: the 18 Kuka values, the 10 final placements (x, y) and the 10 object types
constexpr int KUKA_DIST_DRAWS = 48;
