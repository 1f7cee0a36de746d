// TEST-ONLY: per-instance sampling schedules (InstSchedule, schedule_noise, cta_instance) of
// csrc/dial_device.cuh on the CPU through the lock-step fiber emulator (warp_emul.h), built into its own
// library by tests/test_instance_schedule.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <vector>
#include <string>
#include <stdio.h>
#include "../../dial_mpc_b200/csrc/dial_host.h"

extern "C" size_t emul_sizeof_schedule(void) { return sizeof(InstSchedule); }

// Planner rows (mode 1) of one launch as the control-step graph issues it at diffusion iteration `iter`:
// rows_per_inst rows per instance (0: a single-instance launch), instance-major state / counters / rng /
// knots, the bound noise row `noise` and the schedules `sched` [instances] (nullable).
extern "C" int emul_rollout_schedule(const dial_model_desc* m, const dial_plan_desc* c, int nrows, int H, int rows_per_inst,
                                     int iter, const InstSchedule* sched, const float* qpos0, const float* qvel0,
                                     const float* warm0, const int32_t* counters_in, const uint32_t* rng_dev,
                                     const float* Ybar, const float* noise, float* rews, float* q) {
  static DevModel D;
  static DevPlan P;
  std::string err;
  if (!derive_model(*m, D, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  P.c = *c;
  RolloutArgs A;
  memset(&A, 0, sizeof(A));
  A.nrows = nrows; A.H = H; A.mode = 1; A.rows_per_inst = rows_per_inst;
  A.qpos0 = qpos0; A.qvel0 = qvel0; A.warm0 = warm0; A.counters_in = counters_in; A.rng_dev = rng_dev;
  A.Ybar = Ybar; A.noise = noise; A.sched = sched; A.iter = iter; A.rews = rews; A.q = q;
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

// cta_instance of CTA `cta` for a launch of nrows rows at wpc warps per CTA; with_models: the layout of
// per-instance (rows_per_model = 0) or member (rows_per_model > 0) model slots.
extern "C" int emul_cta_instance(int nrows, int rows_per_inst, int rows_per_model, int with_models, int cta, int wpc) {
  static DevModel slot;
  RolloutArgs A;
  memset(&A, 0, sizeof(A));
  A.nrows = nrows; A.rows_per_inst = rows_per_inst; A.rows_per_model = rows_per_model;
  A.models = with_models ? &slot : nullptr;
  return cta_instance(A, cta, wpc);
}
