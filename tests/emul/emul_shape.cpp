// TEST-ONLY: the star<3,6> rollout specialised on one model's integer structure (ShapeFixed, built with the
// -DDIAL_SHAPE_* values of dial_mpc_b200.modelc.shape) next to the generic one (ShapeRT), on the CPU through
// the lock-step fiber emulator (warp_emul.h); built into its own library by tests/test_emul_shape.py.
// Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <vector>
#include <string>
#include <stdio.h>
#include "../../dial_mpc_b200/csrc/dial_host.h"

#ifndef DIAL_SHAPE_NBODY
#error "compile with the -DDIAL_SHAPE_* values of one shape"
#endif

// 1: a plan of this model + descriptor would launch the specialised kernel (star<3,6> and every fixed
// value equal to its own), 0: the generic one, -1: the model does not derive
extern "C" int emul_shape_selects(const dial_model_desc* m, const dial_plan_desc* c) {
  static DevModel D;
  std::string err;
  if (!derive_model(*m, D, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  return star_variant(D) == 1 && shape_matches<ShapeFixed>(D, *c) ? 1 : 0;
}

// emul_rollout_tasks (emul_tasks.cpp) through the specialised (specialised = 1) or the generic kernel
extern "C" int emul_rollout_shape(int specialised, const dial_model_desc* m, const dial_plan_desc* c,
                                  const dial_task* tasks, int task_rows, int mode, int nrows, int H, int rows_per_inst,
                                  int us_row, const float* qpos0, const float* qvel0, const float* warm0,
                                  const int32_t* counters_in, int32_t* counters_out, const uint32_t* rng_dev,
                                  const float* us, const float* Ybar, const float* noise, float* rewss, float* rews,
                                  float* q, float* qd, float* xpos, float* qpos_out, float* qvel_out,
                                  float* warm_out, float* ctrl_out) {
  static DevModel D;
  static DevPlan P;
  std::string err;
  if (!derive_model(*m, D, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  if (star_variant(D) != 1) { fprintf(stderr, "emul: not a star<3,6> model\n"); return -1; }
  P.c = *c;
  RolloutArgs A;
  memset(&A, 0, sizeof(A));
  A.tasks = tasks; A.task_rows = task_rows;
  A.nrows = nrows; A.H = H; A.mode = mode; A.rows_per_inst = rows_per_inst; A.us_row = us_row;
  A.qpos0 = qpos0; A.qvel0 = qvel0; A.warm0 = warm0; A.counters_in = counters_in; A.counters_out = counters_out;
  A.rng_dev = rng_dev; A.us = us; A.Ybar = Ybar; A.noise = noise; A.rewss = rewss; A.rews = rews; A.q = q; A.qd = qd;
  A.xpos = xpos; A.qpos_out = qpos_out; A.qvel_out = qvel_out; A.warm_out = warm_out; A.ctrl_out = ctrl_out;
  std::vector<float> slab(D.warp_floats, 0.f);
  for (int row = 0; row < nrows; ++row) {
    emul::run_warp([&](int lane) {
      if (specialised) rollout_warp<3, 6, ShapeFixed>(&D, &P, slab.data(), A, row, lane);
      else rollout_warp<3, 6, ShapeRT>(&D, &P, slab.data(), A, row, lane);
    });
  }
  return 0;
}
