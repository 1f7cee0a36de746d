// TEST-ONLY: ensemble rollout launches (dial_plan_desc.n_ens >= 1) of csrc/dial_device.cuh on the CPU
// through the lock-step fiber emulator (warp_emul.h), built into its own library by
// tests/test_ensemble.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <vector>
#include <string>
#include <stdio.h>
#include "../../dial_mpc_b200/csrc/dial_host.h"

// One planner launch (mode 1) of `nrows` rows as dial_mpc_step enqueues it, in CTAs of `wpc` warps mapped
// to rows the way rollout_kernel maps them.  models [n_models] (NULL: the plan's model `m` for every row)
// holds one model per slot of model_rows = rows_per_model, or rows_per_inst when rows_per_model is 0:
// ceil(model_rows / wpc) CTAs per slot, each staging its slot's model, a warp past the slot's last row
// repeating that row.  tasks (nullable) are read per row as tasks[row / task_rows] (tasks[0] when
// task_rows is 0).
extern "C" int emul_rollout_ensemble(const dial_model_desc* m, const dial_model_desc* models, int n_models,
                                     const dial_plan_desc* c, int wpc, int nrows, int H, int rows_per_inst,
                                     int rows_per_model, const dial_task* tasks, int task_rows,
                                     const float* qpos0, const float* qvel0, const float* warm0,
                                     const int32_t* counters_in, const uint32_t* rng_dev, const float* Ybar,
                                     const float* noise, float* rewss, float* rews, float* q, float* qd,
                                     float* xpos) {
  std::string err;
  static DevModel base;
  if (!derive_model(*m, base, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  std::vector<DevModel> gm(models ? n_models : 1, base);
  for (int i = 0; models && i < n_models; ++i) {
    if (!derive_model(models[i], gm[i], err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
    if (const char* d = instance_model_difference(base, gm[i])) { fprintf(stderr, "emul: model %d: %s differs\n", i, d); return -2; }
  }
  static DevPlan P;
  P.c = *c;
  RolloutArgs A;
  memset(&A, 0, sizeof(A));
  A.models = models ? gm.data() : nullptr;
  A.nrows = nrows; A.H = H; A.mode = 1; A.rows_per_inst = rows_per_inst; A.rows_per_model = rows_per_model;
  A.tasks = tasks; A.task_rows = task_rows;
  A.qpos0 = qpos0; A.qvel0 = qvel0; A.warm0 = warm0; A.counters_in = counters_in;
  A.rng_dev = rng_dev; A.Ybar = Ybar; A.noise = noise; A.rewss = rewss; A.rews = rews; A.q = q; A.qd = qd; A.xpos = xpos;
  std::vector<float> slab(base.warp_floats, 0.f);
  const int variant = star_variant(base);
  const int rps = rows_per_model > 0 ? rows_per_model : rows_per_inst;   // model_rows
  const bool slots = A.models && rps > 0;
  const int cpi = slots ? (rps + wpc - 1) / wpc : 0;
  const int grid = slots ? (nrows / rps) * cpi : (nrows + wpc - 1) / wpc;   // launch_rollout's grid
  static DevModel sM;
  for (int cta = 0; cta < grid; ++cta) {
    // the kernel prologue (dial_rollout_variant.cu): the CTA's model slot and the model it stages
    const int slot = slots ? cta / cpi : 0;
    if (slot >= (int)gm.size()) { fprintf(stderr, "emul: CTA %d has no model\n", cta); return -3; }
    sM = gm[slot];
    for (int warp = 0; warp < wpc; ++warp) {
      int row = cta * wpc + warp;
      if (slots) {
        int lrow = (cta - slot * cpi) * wpc + warp;
        if (lrow >= rps) lrow = rps - 1;
        row = slot * rps + lrow;
      }
      if (row >= nrows) row = nrows - 1;
      emul::run_warp([&](int lane) {
        if (variant == 1) rollout_warp<3, 6>(&sM, &P, slab.data(), A, row, lane);
        else if (variant == 2) rollout_warp<5, 7>(&sM, &P, slab.data(), A, row, lane);
        else if (variant == 3) rollout_warp<-1, DIAL_DENSE_NV>(&sM, &P, slab.data(), A, row, lane);
        else if (variant == 4) rollout_warp<5, 6>(&sM, &P, slab.data(), A, row, lane);
        else rollout_warp<0, 0>(&sM, &P, slab.data(), A, row, lane);
      });
    }
  }
  return 0;
}
