// TEST-ONLY: per-instance observation (ObsSetting, ObsRing, observe_advance / observe_record / observe_emit) of
// csrc/dial_device.cuh on the CPU, as observe_kernel runs them with `threads` threads per instance, built into
// its own library by tests/test_instance_observation.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <stdio.h>
#include "../../dial_mpc_b200/csrc/dial_host.h"

extern "C" size_t emul_sizeof_obs(int which) { return which == 0 ? sizeof(ObsSetting) : sizeof(ObsRing); }

// One observe step of one instance: the ring `r` (updated), its records rq [DIAL_OBSRING][nq], rv / rw
// [DIAL_OBSRING][nv], ra [DIAL_OBSRING][nu], rc [DIAL_OBSRING][2]; the plant state and applied action (act
// nullable); the delay d and its pending rows (nullable); out: the observation oq / ov / ow / oc, the planning
// state pq / pv / pw / pc, the prediction's actions seq [DIAL_MAXDELAY][nu], and age / len (len with predict).
// Each of the two stages runs every thread before the next, as the kernel's __syncthreads orders them.
extern "C" int emul_observe_step(const dial_model_desc* m, const ObsSetting* s, ObsRing* r, int env_step, int d,
                                 int predict, const float* pending, const float* qpos, const float* qvel,
                                 const float* warm, const int32_t* cnt, const float* act, float* rq, float* rv,
                                 float* rw, float* ra, int32_t* rc, float* oq, float* ov, float* ow, int32_t* oc,
                                 float* pq, float* pv, float* pw, int32_t* pc, float* seq, int32_t* age,
                                 int32_t* len, int threads) {
  const bool push = observe_pushes(*s, *r, env_step != 0);
  const ObsRing r1 = observe_advance(*s, *r, env_step != 0);
  ObsView V;
  V.qpos = qpos; V.qvel = qvel; V.warm = warm; V.cnt = cnt; V.act = env_step ? act : nullptr;
  V.rq = rq; V.rv = rv; V.rw = rw; V.ra = ra; V.rc = rc;
  V.oq = oq; V.ov = ov; V.ow = ow; V.oc = oc;
  V.pq = pq; V.pv = pv; V.pw = pw; V.pc = pc;
  V.seq = seq; V.pending = pending;
  for (int t = 0; t < threads; ++t) observe_record(push, r1, V, m->nq, m->nv, m->nu, t, threads);
  for (int t = 0; t < threads; ++t) observe_emit(*s, r1, *m, d, V, t, threads);
  *r = r1;
  *age = observe_age(*s, r1);
  *len = predict ? *age + d : 0;
  return 0;
}
