// TEST-ONLY: per-instance pushes (PushTable, push_kinematics / push_rows / push_solve / push_add) of
// csrc/dial_device.cuh on the CPU, as push_kernel runs them with `lanes` lanes per instance, built into its own
// library by tests/test_instance_pushes.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <stdio.h>
#include <string>
#include "../../dial_mpc_b200/csrc/dial_host.h"

extern "C" size_t emul_sizeof_push(int which) { return which == 0 ? sizeof(dial_push) : sizeof(PushTable); }

// One push step of one instance on the model m at post-step counter `step`: returns 1 when some entry fires
// (qvel [nv] updated, dqvel [nv] the fp64 Delta qvel, M [nv][nv] the mass matrix), else 0 with nothing written.
// Each stage runs every lane before the next, as the kernel's __syncwarp orders them.
extern "C" int emul_push_step(const dial_model_desc* m, const PushTable* T, int step, double dt, const float* qpos,
                              float* qvel, double* dqvel, double* M, int lanes) {
  static DevModel D;
  static PushWork W;
  std::string err;
  if (!derive_model(*m, D, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  if (!push_any(*T, step)) return 0;
  const int nv = m->nv;
  push_kinematics(D.m, qpos, W);
  for (int l = 0; l < lanes; ++l) push_rows(D, *T, step, dt, W, l, lanes);
  if (M)
    for (int i = 0; i < nv; ++i)
      for (int j = 0; j < nv; ++j) M[i * nv + j] = W.M[i][j];
  push_solve(nv, W);
  for (int i = 0; i < nv; ++i) {
    if (dqvel) dqvel[i] = W.g[i];
    qvel[i] = push_add(qvel[i], W.g[i]);
  }
  return 1;
}
