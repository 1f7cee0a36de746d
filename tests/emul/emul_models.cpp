// TEST-ONLY: batched rollout launches with per-instance models (dial_plan_set_instance_model) of
// csrc/dial_device.cuh on the CPU through the lock-step fiber emulator (warp_emul.h), built into its own
// library by tests/test_instance_models.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <vector>
#include <string>
#include <stdio.h>
#include "../../dial_mpc_b200/csrc/dial_host.h"

// emul_rollout_batched (emul_batch.cpp) with the model of instance b taken from models[b] (n_models of
// them; NULL: the plan's model `m` for every row), in CTAs of `wpc` warps mapped to rows the way
// rollout_kernel maps them with per-instance models: ceil(rows_per_inst / wpc) CTAs per instance, each
// staging its instance's model, a warp past the instance's last row repeating that row.
extern "C" int emul_rollout_models(const dial_model_desc* m, const dial_model_desc* models, int n_models,
                                   const dial_plan_desc* c, int wpc, int mode, int nrows, int H, int rows_per_inst,
                                   int us_row, const float* qpos0, const float* qvel0, const float* warm0,
                                   const int32_t* counters_in, int32_t* counters_out, const uint32_t* rng_dev,
                                   const float* us, const float* Ybar, const float* noise, float* rewss, float* rews,
                                   float* q, float* qd, float* xpos, float* qpos_out, float* qvel_out,
                                   float* warm_out, float* ctrl_out) {
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
  A.nrows = nrows; A.H = H; A.mode = mode; A.rows_per_inst = rows_per_inst; A.us_row = us_row;
  A.qpos0 = qpos0; A.qvel0 = qvel0; A.warm0 = warm0; A.counters_in = counters_in; A.counters_out = counters_out;
  A.rng_dev = rng_dev; A.us = us; A.Ybar = Ybar; A.noise = noise; A.rewss = rewss; A.rews = rews; A.q = q; A.qd = qd;
  A.xpos = xpos; A.qpos_out = qpos_out; A.qvel_out = qvel_out; A.warm_out = warm_out; A.ctrl_out = ctrl_out;
  std::vector<float> slab(base.warp_floats, 0.f);
  const int variant = star_variant(base);
  const bool per_inst = A.models && rows_per_inst > 0;
  const int cpi = per_inst ? (rows_per_inst + wpc - 1) / wpc : 0;
  const int grid = per_inst ? (nrows / rows_per_inst) * cpi : (nrows + wpc - 1) / wpc;   // launch_rollout's grid
  static DevModel sM;
  for (int cta = 0; cta < grid; ++cta) {
    // the kernel prologue (dial_rollout_variant.cu): the CTA's instance and the model it stages
    const int inst = per_inst ? cta / cpi : 0;
    if (inst >= (int)gm.size()) { fprintf(stderr, "emul: CTA %d has no model\n", cta); return -3; }
    sM = gm[inst];
    for (int warp = 0; warp < wpc; ++warp) {
      int row = cta * wpc + warp;
      if (per_inst) {
        int lrow = (cta - inst * cpi) * wpc + warp;
        if (lrow >= rows_per_inst) lrow = rows_per_inst - 1;
        row = inst * rows_per_inst + lrow;
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

// dial_plan_set_instance_model's check: 0 when `inst` may be an instance model of a plan of `plan`, else
// -1 with the first differing field (or derive_model's error) in `out`.
extern "C" int emul_instance_model_difference(const dial_model_desc* plan, const dial_model_desc* inst, char* out,
                                              int n) {
  static DevModel a, b;
  std::string err;
  const char* d = nullptr;
  if (!derive_model(*plan, a, err) || !derive_model(*inst, b, err)) d = err.c_str();
  else d = instance_model_difference(a, b);
  if (!d) return 0;
  snprintf(out, n, "%s", d);
  return -1;
}
