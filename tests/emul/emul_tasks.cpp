// TEST-ONLY: batched rollout launches with per-instance tasks (dial_mpc_buffers.tasks) of
// csrc/dial_device.cuh on the CPU through the lock-step fiber emulator (warp_emul.h), built into its own
// library by tests/test_emul_tasks.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <vector>
#include <string>
#include <stdio.h>
#include "../../dial_mpc_b200/csrc/dial_host.h"

// emul_rollout_batched (emul_batch.cpp) with the reward inputs of row r read from tasks[r / task_rows],
// as dial_mpc_step launches a plan with bound tasks; tasks == NULL: the plan's own task for every row.
extern "C" int emul_rollout_tasks(const dial_model_desc* m, const dial_plan_desc* c, const dial_task* tasks,
                                  int task_rows, int mode, int nrows, int H, int rows_per_inst, int us_row,
                                  const float* qpos0, const float* qvel0, const float* warm0,
                                  const int32_t* counters_in, int32_t* counters_out, const uint32_t* rng_dev,
                                  const float* us, const float* Ybar, const float* noise, float* rewss, float* rews,
                                  float* q, float* qd, float* xpos, float* qpos_out, float* qvel_out,
                                  float* warm_out, float* ctrl_out) {
  static DevModel D;
  static DevPlan P;
  std::string err;
  if (!derive_model(*m, D, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  P.c = *c;
  RolloutArgs A;
  memset(&A, 0, sizeof(A));
  A.tasks = tasks; A.task_rows = task_rows;
  A.nrows = nrows; A.H = H; A.mode = mode; A.rows_per_inst = rows_per_inst; A.us_row = us_row;
  A.qpos0 = qpos0; A.qvel0 = qvel0; A.warm0 = warm0; A.counters_in = counters_in; A.counters_out = counters_out;
  A.rng_dev = rng_dev; A.us = us; A.Ybar = Ybar; A.noise = noise; A.rewss = rewss; A.rews = rews; A.q = q; A.qd = qd;
  A.xpos = xpos; A.qpos_out = qpos_out; A.qvel_out = qvel_out; A.warm_out = warm_out; A.ctrl_out = ctrl_out;
  std::vector<float> slab(D.warp_floats, 0.f);
  const int variant = star_variant(D);
  for (int row = 0; row < nrows; ++row) {
    emul::run_warp([&](int lane) {
      if (variant == 1) rollout_warp<3, 6>(&D, &P, slab.data(), A, row, lane);
      else if (variant == 2) rollout_warp<5, 7>(&D, &P, slab.data(), A, row, lane);
      else if (variant == 3) rollout_warp<-1, DIAL_DENSE_NV>(&D, &P, slab.data(), A, row, lane);
      else if (variant == 4) rollout_warp<5, 6>(&D, &P, slab.data(), A, row, lane);
      else rollout_warp<0, 0>(&D, &P, slab.data(), A, row, lane);
    });
  }
  return 0;
}
