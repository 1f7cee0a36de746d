// TEST-ONLY: runs the device code of csrc/dial_device.cuh on the CPU, the per-warp code through the
// lock-step fiber emulator (warp_emul.h).  Used by the tests to check kernel logic without a GPU; built by
// tests/emul/emul.py with optional defines (DIAL_TERRAIN, DIAL_SHAPE_*, DIAL_EMUL_TRACE, ...) and custom
// reward.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include <stddef.h>
#include <stdio.h>
#include <string>
#include <vector>
#ifdef DIAL_EMUL_TRACE
static std::vector<int> g_trace;
extern "C" void emul_trace(int kind, int val) { g_trace.push_back(kind); g_trace.push_back(val); }
extern "C" int emul_trace_take(int* out, int cap) {
  int n = (int)g_trace.size() < cap ? (int)g_trace.size() : cap;
  for (int i = 0; i < n; ++i) out[i] = g_trace[i];
  g_trace.clear();
  return n;
}
#endif
#include "../../dial_mpc_b200/csrc/dial_host.h"
#ifdef DIAL_TERRAIN
#include "../../include/dial_custom_reward.h"
#endif

// Every field of RolloutArgs in declaration order: emul.py checks its ctypes mirror against these offsets.
#define ROLLOUT_FIELDS(X)                                                                                      \
  X(nrows) X(H) X(mode) X(lockstep) X(sync_every) X(step0) X(stage0) X(rows_per_inst) X(us_row) X(task_rows) \
  X(tasks) X(qpos0) X(qvel0) X(warm0) X(us) X(eps) X(Ybar) X(noise) X(key0) X(key1) X(rewss) X(rews) X(q)    \
  X(qd) X(xpos) X(qpos_out) X(qvel_out) X(warm_out) X(ctrl_out) X(kin_out) X(counters_in) X(counters_out)    \
  X(key_dev) X(rng_dev) X(row_counter) X(dbg) X(xch_world) X(xch_rank) X(xch_mbox) X(xch_flags) X(xch_seq)   \
  X(xch_done) X(models) X(rows_per_model) X(sched) X(iter_lim) X(iter) X(terrain)

// Field i of RolloutArgs: its name, and its offset in `offset`; past the last field nullptr, and
// sizeof(RolloutArgs) in `offset`.
extern "C" const char* emul_rollout_field(int i, size_t* offset) {
#define NAME(f) #f,
#define OFFSET(f) offsetof(RolloutArgs, f),
  static const char* names[] = {ROLLOUT_FIELDS(NAME)};
  static const size_t offsets[] = {ROLLOUT_FIELDS(OFFSET)};
#undef NAME
#undef OFFSET
  const int n = (int)(sizeof(names) / sizeof(names[0]));
  *offset = i < n ? offsets[i] : sizeof(RolloutArgs);
  return i < n ? names[i] : nullptr;
}

// 0: DelaySetting, 1: ObsSetting, 2: ObsRing, 3: dial_push, 4: PushTable, 5: InstSchedule
extern "C" size_t emul_sizeof(int which) {
  const size_t s[] = {sizeof(DelaySetting), sizeof(ObsSetting), sizeof(ObsRing), sizeof(dial_push),
                      sizeof(PushTable), sizeof(InstSchedule)};
  return which >= 0 && which < 6 ? s[which] : 0;
}

static bool derive(const dial_model_desc& m, DevModel& D) {
  std::string err;
  if (derive_model(m, D, err)) return true;
  fprintf(stderr, "emul: %s\n", err.c_str());
  return false;
}

// derived-model flags (tests): out = {star variant, s_on, sb_on, warp_floats}
extern "C" int emul_model_flags(const dial_model_desc* m, int out[4]) {
  static DevModel D;
  if (!derive(*m, D)) return -1;
  out[0] = star_variant(D); out[1] = D.s_on; out[2] = D.sb_on; out[3] = D.warp_floats;
  return 0;
}

// The prologue of rollout_kernel (dial_rollout_variant.cu), restated for the emulator: the CTAs of a launch
// of `wpc` warps per CTA in order, each exiting whole when its instance is past its iteration limit, else
// staging its model slot (stage(slot)) and running each of its active warps on its row (run(row)).  The
// emulator runs the warps of a CTA one after another, so A.lockstep must be 0: a warp past its slot's or the
// launch's last row idles.  Returns -3 when a CTA's slot is not below n_slots.
template <class Stage, class Run>
static int map_launch(const RolloutArgs& A, int wpc, int n_slots, Stage stage, Run run) {
  const int rps = model_rows(A), grid = rollout_grid(A, wpc);
  const bool slots = A.models && rps > 0;
  const int cpi = slots ? (rps + wpc - 1) / wpc : 0;
  for (int cta = 0; cta < grid; ++cta) {
    if (A.iter_lim && !schedule_runs(A.iter_lim, cta_instance(A, cta, wpc), A.iter)) continue;
    const int slot = slots ? cta / cpi : 0;
    if (slot >= n_slots) { fprintf(stderr, "emul: CTA %d has no model\n", cta); return -3; }
    stage(cta, slot);
    for (int warp = 0; warp < wpc; ++warp) {
      int row = cta * wpc + warp;
      bool active = true;
      if (slots) {
        row = (cta - slot * cpi) * wpc + warp;
        if (row >= rps) {
          active = A.lockstep != 0;
          row = rps - 1;
        }
        row += slot * rps;
      }
      if (row >= A.nrows) {
        active = A.lockstep != 0;
        row = A.nrows - 1;
      }
      if (active) run(row);
    }
  }
  return 0;
}

static DevTerrain dev_terrain(const dial_terrain* t) {
  DevTerrain T;
  memset(&T, 0, sizeof(T));
  if (t) { T.nx = t->nx; T.ny = t->ny; T.x0 = t->x0; T.y0 = t->y0; T.inv = 1.f / t->spacing; T.h = t->heights; }
  return T;
}

// One launch of rollout_kernel as launch_rollout issues it at `wpc` warps per CTA, on the plan model `m` and
// descriptor `c`.  models [n_models] (nullable) are the instance or member models of the launch's model slots,
// terrain [n_terrain] (nullable) its terrain entries; A->models and A->terrain are filled from them.
// kernel: -1 the plan model's solver variant (star_variant), 0..4 that variant, 5 the star<3,6> kernel
// specialised on the DIAL_SHAPE_* values of the build (ShapeFixed).  Returns 0, -1 for a model that does not
// derive (or kernel 5 on another variant or build), -2 for an instance model that differs from the plan's
// beyond its physical parameters, -3 for a CTA without a model.
extern "C" int emul_launch(const dial_model_desc* m, const dial_model_desc* models, int n_models,
                           const dial_plan_desc* c, const dial_terrain* terrain, int n_terrain, RolloutArgs* A,
                           int wpc, int kernel) {
  static DevModel base, sM;
  static DevPlan P;
  if (!derive(*m, base)) return -1;
  std::vector<DevModel> gm(models ? n_models : 0, base);
  for (int i = 0; i < (int)gm.size(); ++i) {
    if (!derive(models[i], gm[i])) return -1;
    if (const char* d = instance_model_difference(base, gm[i])) { fprintf(stderr, "emul: model %d: %s differs\n", i, d); return -2; }
  }
  std::vector<DevTerrain> T(terrain ? n_terrain : 0);
  for (int i = 0; i < (int)T.size(); ++i) T[i] = dev_terrain(terrain + i);
  A->models = models ? gm.data() : nullptr;
  A->terrain = terrain ? T.data() : nullptr;
  P.c = *c;
  const int variant = kernel >= 0 ? kernel : star_variant(base);
#ifdef DIAL_SHAPE_NBODY
  const bool shape_ok = star_variant(base) == 1;
#else
  const bool shape_ok = false;
#endif
  if (variant == 5 && !shape_ok) { fprintf(stderr, "emul: no star<3,6> shape kernel for this model\n"); return -1; }
  std::vector<float> slab(base.warp_floats, 0.f);
  const int rc = map_launch(*A, wpc, models ? n_models : 1,
                            [&](int, int slot) { sM = models ? gm[slot] : base; },
                            [&](int row) {
    emul::run_warp([&](int lane) {
      if (variant == 1) rollout_warp<3, 6>(&sM, &P, slab.data(), *A, row, lane);
      else if (variant == 2) rollout_warp<5, 7>(&sM, &P, slab.data(), *A, row, lane);
      else if (variant == 3) rollout_warp<-1, DIAL_DENSE_NV>(&sM, &P, slab.data(), *A, row, lane);
      else if (variant == 4) rollout_warp<5, 6>(&sM, &P, slab.data(), *A, row, lane);
#ifdef DIAL_SHAPE_NBODY
      else if (variant == 5) rollout_warp<3, 6, ShapeFixed>(&sM, &P, slab.data(), *A, row, lane);
#endif
      else rollout_warp<0, 0>(&sM, &P, slab.data(), *A, row, lane);
    });
  });
  A->models = nullptr;
  A->terrain = nullptr;
  return rc;
}

// emul_launch's CTA and row mapping without the physics: staged[cta] = the slot CTA `cta` stages (-1: it
// exits at entry), runs[row] += 1 for each active warp on `row`.  with_models: the launch has model slots
// (A->models is set to a placeholder).  Returns the grid, or -3 as emul_launch.
extern "C" int emul_launch_map(const RolloutArgs* A0, int with_models, int n_slots, int wpc, int32_t* staged,
                               int32_t* runs) {
  static DevModel slot;
  RolloutArgs A = *A0;
  A.models = with_models ? &slot : nullptr;
  const int grid = rollout_grid(A, wpc);
  for (int i = 0; i < grid; ++i) staged[i] = -1;
  const int rc = map_launch(A, wpc, n_slots, [&](int cta, int s) { staged[cta] = s; }, [&](int row) { runs[row] += 1; });
  return rc < 0 ? rc : grid;
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

// The setting dial_plan_set_ensemble_risk derives: out = {mode, n_tail} and {frac, denom}.
extern "C" void emul_risk_derive(int K, int mode, float alpha, int32_t* iout, float* fout) {
  const EnsRisk R = ens_risk_derive(K, mode, alpha);
  iout[0] = R.mode; iout[1] = R.n_tail; fout[0] = R.frac; fout[1] = R.denom;
}

// The reduction kernel's per-sample work on member rewards r [K][n] (member k of sample i at k n + i).
extern "C" void emul_risk_reduce(const float* r, int K, int n, int mode, float alpha, float* out) {
  const EnsRisk R = ens_risk_derive(K, mode, alpha);
  for (int i = 0; i < n; ++i) out[i] = ens_risk_reduce(r + i, (size_t)n, K, R);
}

// The reduction kernel's per-sample work of an adapting instance: member rewards r [K][n] under the belief w [K].
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

// One observe step of one instance as observe_kernel runs it with `threads` threads: the ring `r` (updated),
// its records rq [DIAL_OBSRING][nq], rv / rw [DIAL_OBSRING][nv], ra [DIAL_OBSRING][nu], rc [DIAL_OBSRING][2];
// the plant state and applied action (act nullable); the delay d and its pending rows (nullable); out: the
// observation oq / ov / ow / oc, the planning state pq / pv / pw / pc, the prediction's actions
// seq [DIAL_MAXDELAY][nu], and age / len (len with predict).  Each of the two stages runs every thread before
// the next, as the kernel's __syncthreads orders them.
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

// One push step of one instance as push_kernel runs it with `lanes` lanes, on the model m at post-step counter
// `step`: returns 1 when some entry fires (qvel [nv] updated, dqvel [nv] the fp64 Delta qvel, M [nv][nv] the
// mass matrix), else 0 with nothing written.  Each stage runs every lane before the next, as the kernel's
// __syncwarp orders them.
extern "C" int emul_push_step(const dial_model_desc* m, const PushTable* T, int step, double dt, const float* qpos,
                              float* qvel, double* dqvel, double* M, int lanes) {
  static DevModel D;
  static PushWork W;
  if (!derive(*m, D)) return -1;
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

#ifdef DIAL_SHAPE_NBODY
// 1: a plan of this model + descriptor would launch the specialised kernel (star<3,6> and every fixed
// value equal to its own), 0: the generic one, -1: the model does not derive
extern "C" int emul_shape_selects(const dial_model_desc* m, const dial_plan_desc* c) {
  static DevModel D;
  if (!derive(*m, D)) return -1;
  return star_variant(D) == 1 && shape_matches<ShapeFixed>(D, *c) ? 1 : 0;
}
#endif

#ifdef DIAL_TERRAIN
// H(x, y) as a custom reward reads it (dial_terrain_height; t NULL: a row without a terrain)
extern "C" float emul_terrain_height(const dial_terrain* t, float x, float y) {
  const DevTerrain T = dev_terrain(t);
  dial_reward_ctx ctx;
  memset(&ctx, 0, sizeof(ctx));
  ctx.terrain = t ? &T : nullptr;
  return dial_terrain_height(&ctx, x, y);
}
#endif
