// TEST-ONLY: the terrain build (-DDIAL_TERRAIN) of csrc/dial_device.cuh on the CPU through the lock-step fiber
// emulator (warp_emul.h): rollouts of one instance on one terrain table, and the surface height a custom reward
// reads.  Built into its own library by tests/test_terrain.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_TERRAIN 1
#include "emul_main.cpp"
#include "../../include/dial_custom_reward.h"

static DevTerrain dev_terrain(const dial_terrain* t) {
  DevTerrain T;
  memset(&T, 0, sizeof(T));
  if (t) { T.nx = t->nx; T.ny = t->ny; T.x0 = t->x0; T.y0 = t->y0; T.inv = 1.f / t->spacing; T.h = t->heights; }
  return T;
}

// emul_rollout with every row on the terrain `t` (NULL: a table whose entry is the flat floor)
extern "C" int emul_rollout_terrain(const dial_model_desc* m, const dial_plan_desc* c, const dial_terrain* t, int mode,
                                    int nrows, int H, int step0, const float* qpos0, const float* qvel0,
                                    const float* warm0, const float* us, float* rewss, float* q, float* qd,
                                    float* qpos_out, float* qvel_out, float* warm_out, float* ctrl_out) {
  static DevModel D;
  static DevPlan P;
  std::string err;
  if (!derive_model(*m, D, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  P.c = *c;
  const DevTerrain T = dev_terrain(t);
  RolloutArgs A;
  memset(&A, 0, sizeof(A));
  A.nrows = nrows; A.H = H; A.mode = mode; A.step0 = step0;
  A.qpos0 = qpos0; A.qvel0 = qvel0; A.warm0 = warm0; A.us = us; A.rewss = rewss; A.q = q; A.qd = qd;
  A.qpos_out = qpos_out; A.qvel_out = qvel_out; A.warm_out = warm_out; A.ctrl_out = ctrl_out;
  A.terrain = &T;
  std::vector<float> slab(D.warp_floats, 0.f);
  const int variant = star_variant(D);
  for (int row = 0; row < nrows; ++row) {
    emul::run_warp([&](int lane) {
      if (variant == 1) rollout_warp<3, 6>(&D, &P, slab.data(), A, row, lane);
      else if (variant == 2) rollout_warp<5, 7>(&D, &P, slab.data(), A, row, lane);
      else if (variant == 4) rollout_warp<5, 6>(&D, &P, slab.data(), A, row, lane);
      else rollout_warp<0, 0>(&D, &P, slab.data(), A, row, lane);
    });
  }
  return 0;
}

// H(x, y) as a custom reward reads it (dial_terrain_height; t NULL: a row without a terrain)
extern "C" float emul_terrain_height(const dial_terrain* t, float x, float y) {
  const DevTerrain T = dev_terrain(t);
  dial_reward_ctx ctx;
  memset(&ctx, 0, sizeof(ctx));
  ctx.terrain = t ? &T : nullptr;
  return dial_terrain_height(&ctx, x, y);
}
