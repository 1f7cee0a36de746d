// TEST-ONLY: per-instance control latency (DelaySetting, delay_queue_step, the prediction launches) of
// csrc/dial_device.cuh on the CPU through the lock-step fiber emulator (warp_emul.h), built into its own
// library by tests/test_instance_delay.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <vector>
#include <string>
#include <stdio.h>
#include "../../dial_mpc_b200/csrc/dial_host.h"

extern "C" size_t emul_sizeof_delay(void) { return sizeof(DelaySetting); }

// One step of an instance's queue as delay_queue_kernel runs it with `threads` threads: each thread t
// passes the elements t, t + threads, ...  Returns the new front slot (every thread's, which must agree).
extern "C" int emul_delay_queue_step(float* ring, int head, int d, int nu, const float* y0, float* applied, float* pending,
                                     int pop, int threads) {
  int h1 = -1;
  for (int t = 0; t < threads; ++t) {
    const int h = delay_queue_step(ring, head, d, nu, y0, applied, pending, pop != 0, t, threads);
    if (h1 >= 0 && h != h1) return -2;
    h1 = h;
  }
  return h1;
}

// One env-step launch (mode 0, H = 1) as dial_mpc_step issues it, CTA by CTA at one warp per CTA, in place on
// the instance-major state and counters: nrows rows, rows_per_inst per instance (0: a single-instance launch),
// action row r at us + r us_row; with iter_lim, the CTAs of an instance with iter >= iter_lim[b] exit at entry
// as rollout_kernel's do (cta_instance).
extern "C" int emul_env_launch(const dial_model_desc* m, const dial_plan_desc* c, int nrows, int rows_per_inst,
                               const float* us, int us_row, const int32_t* iter_lim, int iter, float* qpos, float* qvel,
                               float* warm, int32_t* counters, float* rewss) {
  static DevModel D;
  static DevPlan P;
  std::string err;
  if (!derive_model(*m, D, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  P.c = *c;
  RolloutArgs A;
  memset(&A, 0, sizeof(A));
  A.nrows = nrows; A.H = 1; A.mode = 0; A.rows_per_inst = rows_per_inst; A.us = us; A.us_row = us_row;
  A.iter_lim = iter_lim; A.iter = iter;
  A.qpos0 = qpos; A.qvel0 = qvel; A.warm0 = warm; A.counters_in = counters; A.counters_out = counters;
  A.qpos_out = qpos; A.qvel_out = qvel; A.warm_out = warm; A.rewss = rewss;
  std::vector<float> slab(D.warp_floats, 0.f);
  const int variant = star_variant(D);
  for (int cta = 0; cta < nrows; ++cta) {
    if (A.iter_lim && !schedule_runs(A.iter_lim, cta_instance(A, cta, 1), A.iter)) continue;
    emul::run_warp([&](int lane) {
      if (variant == 1) rollout_warp<3, 6>(&D, &P, slab.data(), A, cta, lane);
      else if (variant == 2) rollout_warp<5, 7>(&D, &P, slab.data(), A, cta, lane);
      else if (variant == 3) rollout_warp<-1, DIAL_DENSE_NV>(&D, &P, slab.data(), A, cta, lane);
      else if (variant == 4) rollout_warp<5, 6>(&D, &P, slab.data(), A, cta, lane);
      else rollout_warp<0, 0>(&D, &P, slab.data(), A, cta, lane);
    });
  }
  return 0;
}
