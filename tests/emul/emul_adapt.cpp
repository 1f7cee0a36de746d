// TEST-ONLY: adapting an ensemble plan to its plant (csrc/dial_device.cuh: ens_member_loglik and
// ens_belief_update in ens_belief_kernel, ens_risk_reduce_weighted in the reduction kernel, and the
// member-prediction rollout launch of mpc_enqueue) compiled by g++ with -ffp-contract=off, so that the _rn
// intrinsic shims of the emulator build round each operation as the GPU does.  Built into its own library
// by tests/test_ensemble_adapt.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <vector>
#include <string>
#include <stdio.h>
#include "../../dial_mpc_b200/csrc/dial_host.h"

// The reduction kernel's per-sample work of an adapting instance: member rewards r [K][n] (member k of
// sample i at k n + i) under the belief w [K].
extern "C" void emul_adapt_reduce(const float* r, int K, int n, int mode, float alpha, const float* w, float prune,
                                  float* out) {
  const EnsRisk R = ens_risk_derive(K, mode, alpha);
  for (int i = 0; i < n; ++i) out[i] = ens_risk_reduce_weighted(r + i, (size_t)n, K, R, w, prune);
}

// The belief kernel's work on one instance: l_k from the predictions vhat [K][nv], then the update of
// L [K] in place; w [K] and ell [K] out.
extern "C" void emul_adapt_update(const float* vhat, const float* v, const float* sigma, int K, int nv, float forget,
                                  double* L, float* w, double* ell) {
  for (int k = 0; k < K; ++k) ell[k] = ens_member_loglik(vhat + (size_t)k * nv, v, sigma, nv);
  ens_belief_update(L, w, ell, K, (double)forget);
}

// One env-step launch (mode 0, H = 1, one warp per CTA) of nrows rows as launch_rollout maps them:
// models [n_models] (NULL: the model `m` for every row) holds one model per slot of model_rows =
// rows_per_model, or rows_per_inst when rows_per_model is 0; state, counters and task of row r come from
// instance r / rows_per_inst (0 when rows_per_inst is 0).  The per-row qvel goes to qd [nrows][nv] and the
// final state of each instance's first row to qvel_out [instances][nv] (either nullable).
extern "C" int emul_env_step_rows(const dial_model_desc* m, const dial_model_desc* models, int n_models,
                                  const dial_plan_desc* c, int nrows, int rows_per_inst, int rows_per_model,
                                  const dial_task* tasks, int task_rows, const float* qpos0, const float* qvel0,
                                  const float* warm0, const int32_t* counters_in, const float* us, float* qd,
                                  float* qvel_out) {
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
  A.nrows = nrows; A.H = 1; A.mode = 0; A.rows_per_inst = rows_per_inst; A.rows_per_model = rows_per_model;
  A.tasks = tasks; A.task_rows = task_rows;
  A.qpos0 = qpos0; A.qvel0 = qvel0; A.warm0 = warm0; A.counters_in = counters_in; A.us = us;
  A.qd = qd; A.qvel_out = qvel_out;
  std::vector<float> slab(base.warp_floats, 0.f);
  const int variant = star_variant(base);
  const int rps = rows_per_model > 0 ? rows_per_model : rows_per_inst;   // model_rows
  const bool slots = A.models && rps > 0;
  static DevModel sM;
  for (int row = 0; row < nrows; ++row) {   // one warp per CTA: CTA `row` holds row `row`
    const int slot = slots ? row / rps : 0;
    if (slot >= (int)gm.size()) { fprintf(stderr, "emul: row %d has no model\n", row); return -3; }
    sM = gm[slot];
    emul::run_warp([&](int lane) {
      if (variant == 1) rollout_warp<3, 6>(&sM, &P, slab.data(), A, row, lane);
      else if (variant == 2) rollout_warp<5, 7>(&sM, &P, slab.data(), A, row, lane);
      else if (variant == 3) rollout_warp<-1, DIAL_DENSE_NV>(&sM, &P, slab.data(), A, row, lane);
      else if (variant == 4) rollout_warp<5, 6>(&sM, &P, slab.data(), A, row, lane);
      else rollout_warp<0, 0>(&sM, &P, slab.data(), A, row, lane);
    });
  }
  return 0;
}
