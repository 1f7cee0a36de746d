/*
 * dial_custom_reward.h — device-side contract of a user-written reward
 * (DIAL_ENV_CUSTOM).
 *
 * The reference lets users subclass `BaseEnv` and write `step`/`reset` in JAX
 * (README.md:223-312, `--custom-env` at core/dial_core.py:202-204).  Here the physics of
 * `step` is the fused rollout kernel; the user supplies only the reward as ONE device
 * function in a `.cuh` file,
 *
 *     DIAL_REWARD_FN float dial_custom_reward(const dial_reward_ctx* c);
 *
 * and `dial_mpc_b200.custom.build_library(path)` compiles a dedicated build of
 * libdial_b200 with `-DDIAL_CUSTOM_REWARD_FILE=<path>`.  The function runs on one lane of the
 * warp that owns the sample, once per env step, right after the `n_frames` physics substeps
 * — the place of the reward block in the reference envs (e.g. envs/unitree_go2_env.py:140-235).
 * All pointers address the warp's shared-memory slab (read-only for the reward) or the
 * plan constants; nothing may be kept across calls.
 *
 * What the fields hold (same staleness as Brax's `pipeline_step`: kinematic quantities are
 * those `mjx.step` computed BEFORE integrating, `qpos`/`qvel` are the integrated state):
 */
#ifndef DIAL_CUSTOM_REWARD_H_
#define DIAL_CUSTOM_REWARD_H_

#if defined(__CUDACC__)
#define DIAL_REWARD_FN __device__ __forceinline__
#else
#define DIAL_REWARD_FN inline /* host build of the test-only warp emulator */
#endif

typedef struct dial_reward_ctx {
  int step;           /* state.info["step"] BEFORE the increment (reference reward code reads it so) */
  float dt;           /* env dt = n_frames * timestep                                  */
  int nq, nv, nu, nbody, ncon, nsite, n_user;
  const float* qpos;  /* [nq]  pipeline_state.qpos (after the step)                    */
  const float* qvel;  /* [nv]  pipeline_state.qvel                                     */
  const float* ctrl;  /* [nu]  applied control (torque, or position target)            */
  const float* xpos;  /* [nbody][3] world position of body frames; Brax x.pos[i] = xpos[i+1] */
  const float* xquat; /* [nbody][4] (w,x,y,z);                  Brax x.rot[i] = xquat[i+1]   */
  const float* xmat;  /* [nbody][9] row-major rotation matrices                        */
  const float* cvel;  /* [nbody][6] MuJoCo cvel (ang, lin) in the subtree-COM frame    */
  const float* subtree_com; /* [nroot][3] COM of each kinematic tree (frame of cvel)   */
  const int* body_rootidx;  /* [nbody] index into subtree_com                          */
  const float* contact_dist; /* [ncon] pipeline_state.contact.dist                     */
  const float* contact_pos;  /* [ncon][3] pipeline_state.contact.pos                   */
  const int* site_bodyid;    /* [nsite]                                                */
  const float* site_pos;     /* [nsite][3] site offsets in their body frame            */
  const float* user;         /* [n_user] dial_plan_desc.user                           */
  const void* terrain;       /* this row's terrain (read it with dial_terrain_height)  */
} dial_reward_ctx;

/* Brax xd.ang[body-1]: world angular velocity (rad/s) */
DIAL_REWARD_FN void dial_xd_ang(const dial_reward_ctx* c, int body, float out[3]) {
  const float* v = c->cvel + 6 * body;
  out[0] = v[0]; out[1] = v[1]; out[2] = v[2];
}

/* Brax xd.vel[body-1]: world linear velocity of the body-frame origin
 * (brax.mjx.pipeline: cvel transported from the subtree COM to x.pos) */
DIAL_REWARD_FN void dial_xd_vel(const dial_reward_ctx* c, int body, float out[3]) {
  const float* v = c->cvel + 6 * body;
  const float* p = c->xpos + 3 * body;
  const float* r = c->subtree_com + 3 * c->body_rootidx[body];
  const float ox = p[0] - r[0], oy = p[1] - r[1], oz = p[2] - r[2];
  out[0] = v[3] - (oy * v[2] - oz * v[1]);
  out[1] = v[4] - (oz * v[0] - ox * v[2]);
  out[2] = v[5] - (ox * v[1] - oy * v[0]);
}

/* pipeline_state.site_xpos[site] */
DIAL_REWARD_FN void dial_site_xpos(const dial_reward_ctx* c, int site, float out[3]) {
  const int b = c->site_bodyid[site];
  const float* X = c->xmat + 9 * b;
  const float* s = c->site_pos + 3 * site;
  const float* p = c->xpos + 3 * b;
  out[0] = p[0] + X[0] * s[0] + X[1] * s[1] + X[2] * s[2];
  out[1] = p[1] + X[3] * s[0] + X[4] * s[1] + X[5] * s[2];
  out[2] = p[2] + X[6] * s[0] + X[7] * s[1] + X[8] * s[2];
}

/* Height H(x, y) of the terrain beneath the world point (x, y) on this row (include/dial_b200.h,
 * dial_plan_set_instance_terrain); 0 on a row without a terrain.  Lets a reward measure heights above the
 * ground. */
DIAL_REWARD_FN float dial_terrain_height(const dial_reward_ctx* c, float x, float y) {
  return terrain_height(c->terrain, x, y);
}

#endif /* DIAL_CUSTOM_REWARD_H_ */
