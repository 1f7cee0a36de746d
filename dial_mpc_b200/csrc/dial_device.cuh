// dial_device.cuh — per-warp device code of the DIAL-MPC sampling core (sm_90a).
//
// One warp owns one sample for the whole horizon ("persistent" over Hsample+1 env
// steps): generalized state, the inertia tree and every intermediate of the
// rigid-body step live in a per-warp slab of shared memory / registers; HBM is
// touched only for the per-step outputs (reward, q, qd, x.pos).  Lanes map to
// bodies (kinematics, tree passes), dofs (mass-matrix rows, vectors) or constraint
// rows (contact pyramid edges), whichever the phase needs.
//
// The physics restates mjx.step (third party; reached by the reference through
// brax PipelineEnv.pipeline_step, dial_mpc/envs/unitree_go2_env.py:135) in fp32:
// kinematics -> COM frame (cinert, cdof) -> CRB mass matrix -> collision ->
// constraint rows -> velocity/RNE bias -> actuation -> Newton solve -> Euler.
//
// The file is also compiled by g++ with -DDIAL_HOST_EMUL (tests/emul) where a warp
// is emulated by 32 lock-step fibers; that build exists only to debug kernel logic
// on machines without a GPU and is never used by the product path.
#pragma once

#include <stdint.h>
#include <math.h>
#include "../../include/dial_b200.h"

#ifdef DIAL_HOST_EMUL
#include "warp_emul.h"
#define DEV inline
#define HD inline
// the emulator does not model the GPU's fused multiply-adds: a pinned one rounds as the unpinned code does there
inline float __fmaf_rn(float a, float b, float c) { return a * b + c; }
// IEEE single operations with round-to-nearest (build with -ffp-contract=off so none is fused)
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dsub_rn(double a, double b) { return a - b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __ddiv_rn(double a, double b) { return a / b; }
#else
#define HD __host__ __device__ __forceinline__
#define DEV __device__ __forceinline__
DEV void syncwarp() { __syncwarp(); }
DEV float shfl(float v, int src) { return __shfl_sync(0xffffffffu, v, src); }
DEV float shfl_xor(float v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
DEV int shfl_i(int v, int src) { return __shfl_sync(0xffffffffu, v, src); }
DEV void cta_sync() { __syncthreads(); }
DEV bool cta_sync_or(bool p) { return __syncthreads_or(p) != 0; }
DEV void fast_sincos(float x, float& s, float& c) { __sincosf(x, &s, &c); }
DEV float fast_cos(float x) { return __cosf(x); }
#endif
#ifdef DIAL_HOST_EMUL
inline float ldg(const float* p) { return *p; }
#else
DEV float ldg(const float* p) { return __ldg(p); }   // the read-only data path
#endif

// TEST-ONLY (emulator build with -DDIAL_EMUL_TRACE): iteration counts of the solvers
#if defined(DIAL_HOST_EMUL) && defined(DIAL_EMUL_TRACE)
extern "C" void emul_trace(int kind, int val);
#define DIAL_TRACE(lane, kind, val) do { if ((lane) == 0) emul_trace(kind, val); } while (0)
#else
#define DIAL_TRACE(lane, kind, val) do { } while (0)
#endif

#define DIAL_MAXCHAIN 12   // longest dof ancestor chain (H1: 6 + 5 = 11)
#define DIAL_MAXLEVEL 28
#define DIAL_MAXE 32       // contact pyramid edge rows (4 per contact)
#define DIAL_MINVAL 1e-15f
#define DIAL_MINIMP 1e-4f
#define DIAL_MAXIMP 0.9999f

enum { JNT_FREE = 0, JNT_BALL = 1, JNT_SLIDE = 2, JNT_HINGE = 3 };
enum { PAIR_PLANE_SPHERE = 0, PAIR_PLANE_CAPSULE = 1, PAIR_SPHERE_SPHERE = 2, PAIR_SPHERE_CAPSULE = 3, PAIR_CAPSULE_CAPSULE = 4 };

// ---------------------------------------------------------------------------------
// device-side model: the C-ABI descriptor + host-derived schedules + smem offsets
// ---------------------------------------------------------------------------------
struct alignas(16) DevModel {
  dial_model_desc m;
  // derived on the host (dial_capi.cu: derive_model)
  int32_t maxdepth;
  int32_t nroot, root_body[4];
  float root_invmass[4];
  int32_t body_rootidx[DIAL_MAXB];
  int32_t body_ndesc[DIAL_MAXB];      // descendant bodies (contiguous after b: depth-first order)
  int32_t dof_level[DIAL_MAXV], nlevel;
  int32_t level_adr[DIAL_MAXLEVEL + 1], level_dofs[DIAL_MAXV];
  uint32_t dof_ancmask[DIAL_MAXV];    // bit j: dof j is ancestor-or-self of dof i
  uint32_t body_dofmask[DIAL_MAXB];   // bit d: dof d moves body b
  int32_t dof_actuator[DIAL_MAXV];    // actuator driving the dof or -1
  int32_t dof_limited[DIAL_MAXV];     // joint id if the dof's joint is limited else -1
  int32_t con_pair[DIAL_MAXC], con_sub[DIAL_MAXC];
  int32_t dense;                      // 1: dense / elliptic solver path (NL < 0)
  int32_t con_row0[DIAL_MAXC], con_dim[DIAL_MAXC], nrow_c;
  // dense path: a contact row is non-zero only at the dofs that move exactly one of its two
  // bodies, so J rows are stored with `jd_stride` packed columns; con_colidx[c][d] = packed
  // column of dof d in the rows of contact c, or -1 (structural zero)
  int32_t jd_stride;
  int8_t con_colidx[DIAL_MAXC][DIAL_MAXV];
  int32_t con_lastdof[DIAL_MAXC];     // deepest dof moving the contact's body (geom1 must be static)
  int32_t dof_nchain[DIAL_MAXV], dof_ndesc[DIAL_MAXV], nlimited;
  int32_t chain_tab[DIAL_MAXV][DIAL_MAXCHAIN];
  // star decomposition: root chain + hanging serial chains (0 chains: not a star)
  int32_t star_nroot, star_nchain, star_maxlen;
  int32_t star_root[8], star_len[4], star_leaf[4], star_att[4];
  int32_t nedge;                      // 4 * ncon
  // "star layout" of the solver matrices (star variants only, see the star_* functions): dofs are
  // renumbered root chain first (NRP = NR rounded up to 4 slots), then each hanging chain in a slot
  // of CS = NL rounded up to 4; a row of M / H / J is [NRP root columns | CS columns of its own chain]
  int32_t s_on, s_nrp, s_cs, s_rs, s_npos;
  int32_t s_pos[DIAL_MAXV];           // star position of a dof
  int32_t s_chain[DIAL_MAXV];         // chain of a dof, -1: root dof
  int32_t s_depth[DIAL_MAXV];         // depth inside its chain (0 = attached to the root chain) / root index a (0 = deepest)
  int32_t s_top[4];                   // first (top) dof of chain l; its dofs are s_top[l] + depth (depth-first order)
  int32_t s_con_chain[DIAL_MAXC];     // chain that moves the contact body (-1: root dofs only)
  int32_t o_Ms, o_Hs, o_Js, o_xs;     // star-layout scratch (overlays Mb / L / J / xch)
  // the same star at body level (subtree sums): root bodies (deepest first) + one contiguous run of
  // bodies per hanging chain; sb_on = 0: some body is outside this pattern (welded bodies, ...)
  int32_t sb_on, sb_nroot, sb_root[4], sb_top[4], sb_len[4], sb_att[4];
  // per-warp shared-memory layout (float offsets)
  int32_t o_xpos, o_xquat, o_xmat, o_xipos, o_cinert, o_cdof, o_cdofdot, o_cvel, o_cacc,
      o_cfrc, o_Mb, o_L, o_J, o_qpos, o_qvel, o_warm, o_ctrl, o_vec, o_frow, o_cpos,
      o_cframe, o_cdist, o_rcom, o_xch, o_crb, o_cfs, o_Md, o_Ld, o_Jd, o_Gd, o_frow2, o_cact, o_hcs, warp_floats;
  int32_t pad_[1];
};

struct alignas(16) DevPlan {
  dial_plan_desc c;
  int32_t pad_[3];
};

// The block vel_cmd .. user of dial_plan_desc has the layout of dial_task (include/dial_b200.h): a
// launch without per-instance tasks reads the plan's own task through a view of it.
#define DIAL_TASK_AT(f) (offsetof(dial_plan_desc, f) - offsetof(dial_plan_desc, vel_cmd) == offsetof(dial_task, f))
static_assert(DIAL_TASK_AT(vel_cmd) && DIAL_TASK_AT(ang_cmd) && DIAL_TASK_AT(pos_tar) && DIAL_TASK_AT(gait_duty) &&
              DIAL_TASK_AT(gait_cadence) && DIAL_TASK_AT(gait_amplitude) && DIAL_TASK_AT(gait_phase) &&
              DIAL_TASK_AT(cmd_step) && DIAL_TASK_AT(cmd_vel) && DIAL_TASK_AT(cmd_ang) && DIAL_TASK_AT(n_stage) &&
              DIAL_TASK_AT(jump_dt) && DIAL_TASK_AT(pose_seq) && DIAL_TASK_AT(yaw_seq) &&
              DIAL_TASK_AT(contact_targets) && DIAL_TASK_AT(contact_radius) && DIAL_TASK_AT(n_user) &&
              DIAL_TASK_AT(user) &&
              offsetof(dial_plan_desc, user) + sizeof(float) * DIAL_MAXUSER - offsetof(dial_plan_desc, vel_cmd) == sizeof(dial_task),
              "dial_plan_desc's task block must have the layout of dial_task");
#undef DIAL_TASK_AT

HD const dial_task& plan_task(const dial_plan_desc& c) { return *reinterpret_cast<const dial_task*>(c.vel_cmd); }

// Instance b's own sampling schedule (dial_plan_set_instance_schedule): while `on`, its rollout rows and
// its update take noise row `iter` of its table and its temperature instead of the bound noise and the
// plan's temp_sample.
struct alignas(16) InstSchedule {
  int32_t on;
  float temp;
  int32_t n_rows;   // rows of `noise` set (1..DIAL_MAXDIFFUSE)
  int32_t pad;
  float noise[DIAL_MAXDIFFUSE][DIAL_MAXNODE];
};
// the noise row of instance `inst` at diffusion iteration `iter`: its own, or `bound` (the plan's row)
HD const float* schedule_noise(const InstSchedule* S, int inst, int iter, const float* bound) {
  return (S && S[inst].on) ? S[inst].noise[iter] : bound;
}
// instance `inst` runs diffusion iteration `iter` of a control step (dial_plan_set_instance_iterations;
// no limits: every instance runs every iteration)
HD bool schedule_runs(const int32_t* lim, int inst, int iter) { return !lim || iter < lim[inst]; }

// Instance b's control latency (dial_plan_set_instance_delay): d control steps, and whether it plans from
// the state predicted through its queued actions.
struct alignas(8) DelaySetting {
  int32_t d;         // 0..DIAL_MAXDELAY
  int32_t predict;   // 0 or 1
};
// The action queue of one instance is a ring of d slots of nu floats whose front is slot `head`.  Position
// i of the queue (0: the front, applied next) is slot delay_slot(head, d, i).
HD int delay_slot(int head, int d, int i) { const int s = head + i; return s >= d ? s - d : s; }
// One control step of the queue, for the action elements a = a0, a0 + da, ... < nu (a CTA passes its
// threads).  pop (a step with an env step): applied[a] = the front's element (y0[a] when d = 0), and y0[a]
// takes the front's slot, which becomes the back.  Then, always: pending [DIAL_MAXDELAY][nu] = the queue in
// application order, zero past d.  Returns the front slot after the step.  Each element is read and
// written by one caller only, so callers that split the elements need no synchronisation.
DEV int delay_queue_step(float* ring, int head, int d, int nu, const float* y0, float* applied, float* pending,
                         bool pop, int a0, int da) {
  const int h1 = pop && d > 0 ? delay_slot(head, d, 1) : head;
  for (int a = a0; a < nu; a += da) {
    if (pop) {
      if (d == 0) {
        applied[a] = y0[a];
      } else {
        applied[a] = ring[head * nu + a];
        ring[head * nu + a] = y0[a];
      }
    }
    for (int j = 0; j < DIAL_MAXDELAY; ++j) pending[j * nu + a] = j < d ? ring[delay_slot(h1, d, j) * nu + a] : 0.f;
  }
  return h1;
}

// One instance's terrain on one side (dial_plan_set_instance_terrain, include/dial_b200.h): nx == 0 is the flat
// floor.  `inv` = 1 / spacing; h [ny][nx] is plan-owned device memory.
struct alignas(16) DevTerrain {
  int32_t nx, ny;
  float x0, y0, inv, pad_;
  const float* h;
};

// The plane of the terrain's surface under (x, y): returns its height H(x, y) there and the slopes (sx, sy) of
// the triangle beneath.  Outside the grid the point is clamped into it and the plane is horizontal.  Three
// loads through the read-only path.
DEV float terrain_at(const DevTerrain& T, float x, float y, float& sx, float& sy) {
  const float gx = (float)(T.nx - 1), gy = (float)(T.ny - 1);
  float u = (x - T.x0) * T.inv, v = (y - T.y0) * T.inv;
  const bool inside = u >= 0.f && u <= gx && v >= 0.f && v <= gy;   // (false for NaN)
  u = fminf(fmaxf(u, 0.f), gx); v = fminf(fmaxf(v, 0.f), gy);        // (NaN -> 0)
  const int i = (int)u < T.nx - 2 ? (int)u : T.nx - 2, j = (int)v < T.ny - 2 ? (int)v : T.ny - 2;
  const float fu = u - (float)i, fv = v - (float)j;
  const float* h = T.h + (size_t)j * T.nx + i;
  // the cell's diagonal runs from (i, j) to (i+1, j+1): below it the triangle (i, j), (i+1, j), (i+1, j+1),
  // above it (i, j), (i, j+1), (i+1, j+1); hm is the height of the triangle's third vertex
  const bool lower = fu >= fv;
  const float h00 = ldg(h), h11 = ldg(h + T.nx + 1), hm = ldg(lower ? h + 1 : h + T.nx);
  const float a = lower ? hm - h00 : h11 - hm, b = lower ? h11 - hm : hm - h00;   // rise per cell along x, y
  sx = inside ? a * T.inv : 0.f;
  sy = inside ? b * T.inv : 0.f;
  return h00 + fu * a + fv * b;
}
// H(x, y) of a terrain descriptor, 0 for none or the flat floor (dial_terrain_height of a custom reward)
DEV float terrain_height(const void* t, float x, float y) {
  const DevTerrain* T = static_cast<const DevTerrain*>(t);
  float sx, sy;
  return T && T->nx > 0 ? terrain_at(*T, x, y, sx, sy) : 0.f;
}

// arguments of one rollout launch
struct RolloutArgs {
  int32_t nrows;        // sample rows rolled by this launch
  int32_t H;            // env steps per row
  int32_t mode;         // 0: explicit us; 1: planner (Y0s from eps / key); 2: forward only (pipeline_init)
  int32_t lockstep;     // >=1: warps of a CTA re-converge at every env step (shared instruction fetch); 2: and before the Newton loop
  int32_t sync_every;   // lock-step barrier every this many env steps (>= 1)
  int32_t step0, stage0;
  // batched plans (dial_plan_desc.n_inst > 1): rows [b * rows_per_inst, (b+1) * rows_per_inst) belong to
  // instance b, whose state / counters / rng / key / Ybar and final-state outputs sit at instance-major
  // offsets of the pointers below; per-row outputs are indexed by the global row.  0: one instance.
  int32_t rows_per_inst;
  int32_t us_row;       // floats between the action rows of `us` (mode 0); 0: H * nu
  // per-instance reward inputs (dial_mpc_buffers.tasks): row r reads tasks[r / task_rows], or tasks[0]
  // for every row when task_rows == 0; null: every row reads the plan's own task (plan_task)
  int32_t task_rows;
  const dial_task* tasks;
  const float* qpos0;
  const float* qvel0;
  const float* warm0;
  const float* us;      // [nrows,H,nu]               (mode 0), rows us_row floats apart
  const float* eps;     // [Ntotal,Hn+1,nu] or null   (mode 1)
  const float* Ybar;    // [Hn+1,nu]
  const float* noise;   // [Hn+1]
  uint32_t key0, key1;
  float* rewss;         // [nrows,H] or null
  float* rews;          // [nrows] mean over H or null
  float* q;             // [nrows,H,nq] or null
  float* qd;            // [nrows,H,nv] or null
  float* xpos;          // [nrows,H,nbody-1,3] or null
  float* qpos_out;      // final state of row 0 (env_step / pipeline_init) or null
  float* qvel_out;
  float* warm_out;
  float* ctrl_out;
  float* kin_out;       // [13] x.pos(3), x.rot(4), body-frame xd.vel(3), xd.ang*pi/180(3) of the torso body after row 0's last step, or null
  // device-resident MPC loop (dial_mpc_step): counters / key live in HBM so that a captured CUDA
  // graph can be replayed without patching kernel arguments
  const int32_t* counters_in;   // non-null: {step0, stage0} read from here
  int32_t* counters_out;        // non-null: row 0 writes {step, stage} after its H steps
  const uint32_t* key_dev;      // non-null: sampling key read from here
  const uint32_t* rng_dev;      // non-null: planner rng; the sampling key is split(rng)[1] (the update kernel advances rng)
  unsigned int* row_counter;  // non-null: persistent warps pull rows from this counter (dense path)
  float* dbg;           // optional device counters (DIAL_DEBUG_COUNTERS, see dial_debug_counters)
  // multi-GPU reward exchange fused into the epilogue (dial_exchange_*): every finished row stores
  // its mean reward straight into the mailbox of EVERY rank over NVLink peer memory; the last CTA
  // of the grid then raises this rank's flag in every mailbox.  xch_world <= 1: off.
  int32_t xch_world, xch_rank;
  float* xch_mbox[DIAL_MAXRANK];         // mailbox of rank p: [2][Ntotal+1] floats (double-buffered by sequence parity)
  uint32_t* xch_flags[DIAL_MAXRANK];     // flags of rank p:   [2][DIAL_MAXRANK], slot [buf][source rank] = sequence + 1
  const uint32_t* xch_seq;               // local: sequence number of the current reverse_once
  unsigned int* xch_done;                // local: CTAs of this launch that have finished
  // per-instance models (dial_plan_set_instance_model), [instances] or null: row r runs the model of
  // instance r / rows_per_inst (models[0] when rows_per_inst == 0).  The grid then has
  // ceil(rows_per_inst / blockDim-warps) CTAs per instance, each staging its instance's model.
  const DevModel* models;
  // ensemble plans (dial_plan_desc.n_ens >= 1): the rows of instance b are K member blocks of
  // rows_per_model = Nsample+1 rows each (rows_per_inst = K * rows_per_model); a member's row i takes
  // sample i's perturbation, and `models` holds one model per member block.  0: one block per instance.
  int32_t rows_per_model;
  // per-instance sampling schedules (mode 1 of dial_mpc_step): `iter` is the diffusion iteration of the
  // launch; `sched` [instances] or null (schedule_noise); `iter_lim` [instances] or null: the rows of
  // instance b run only while iter < iter_lim[b], so the host then launches instance-aligned CTAs (the
  // layout of `models`) and a skipped instance's CTAs exit whole (cta_instance)
  const InstSchedule* sched;
  const int32_t* iter_lim;
  int32_t iter;
  // per-instance terrain (dial_plan_set_instance_terrain), [instances] or null: row r reads entry
  // r / rows_per_inst (entry 0 when rows_per_inst == 0); nx == 0 is the flat floor.  Read by the terrain
  // builds (-DDIAL_TERRAIN) only.
  const DevTerrain* terrain;
};

// rows of one model slot of `models`: a member block of an ensemble plan, else an instance
HD int model_rows(const RolloutArgs& A) { return A.rows_per_model > 0 ? A.rows_per_model : A.rows_per_inst; }

// The instance every row of CTA `cta` belongs to under rollout_kernel's row mapping for `wpc` warps per
// CTA, or -1 when the CTA's rows straddle two instances (possible only without `models`).  With `models`
// a CTA holds rows of one model slot: slot s of an ensemble plan is member s % K of instance s / K.
HD int cta_instance(const RolloutArgs& A, int cta, int wpc) {
  if (A.rows_per_inst <= 0) return 0;
  if (A.models && model_rows(A) > 0) {
    const int rps = model_rows(A), slot = cta / ((rps + wpc - 1) / wpc);
    return (int)((int64_t)slot * rps / A.rows_per_inst);
  }
  const int r0 = cta * wpc, r1 = (r0 + wpc < A.nrows ? r0 + wpc : A.nrows) - 1;
  return r0 / A.rows_per_inst == r1 / A.rows_per_inst ? r0 / A.rows_per_inst : -1;
}

// The CTAs of a rollout_kernel launch at `wpc` warps per CTA: one per wpc rows, or with `models`
// ceil(model_rows / wpc) per model slot (the kernel's row mapping)
HD int rollout_grid(const RolloutArgs& A, int wpc) {
  if (A.models && model_rows(A) > 0) return (A.nrows / model_rows(A)) * ((model_rows(A) + wpc - 1) / wpc);
  return (A.nrows + wpc - 1) / wpc;
}

// ---------------------------------------------------------------------------------
// Risk measure of an ensemble plan (dial_plan_set_ensemble_risk): how the K >= 2 member rewards of one
// sample become its score.  The host derives the setting once (ens_risk_derive); the reduction kernel
// (dial_kernels.cu) applies it per (instance, sample) with ens_risk_reduce, which the emulator build
// also runs on the CPU.
// ---------------------------------------------------------------------------------
struct alignas(16) EnsRisk {
  int32_t mode;     // DIAL_ENS_MEAN or DIAL_ENS_CVAR
  int32_t n_tail;   // CVaR: the n_tail lowest rewards count in full
  float frac;       // CVaR: the weight of the next-lowest reward s_{n_tail} (0: none)
  float denom;      // CVaR: the divisor (alpha K; n_tail when frac == 0)
  // read by the belief-weighted branches only (ens_risk_reduce_weighted)
  float alpha;      // CVaR: the fraction of the belief's mass averaged
  int32_t worst;    // CVaR with alpha K <= 1 + 1e-6: the minimum
  int32_t pad_[2];
};

// (K, mode, alpha) -> the setting, in fp64 (include/dial_b200.h: dial_plan_set_ensemble_risk)
inline EnsRisk ens_risk_derive(int K, int mode, float alpha) {
  EnsRisk R;
  R.mode = mode; R.n_tail = K; R.frac = 0.f; R.denom = (float)K;
  R.alpha = 1.f; R.worst = 0; R.pad_[0] = R.pad_[1] = 0;
  if (mode != DIAL_ENS_CVAR) return R;
  R.alpha = alpha;
  const double t = (double)alpha * K;
  if (t <= 1.0 + 1e-6) { R.n_tail = 1; R.denom = 1.f; R.worst = 1; }          // the worst case: the minimum
  else if (fabs(t - round(t)) <= 1e-6 * K) { R.n_tail = (int)round(t); R.denom = (float)R.n_tail; }
  else { R.n_tail = (int)floor(t); R.frac = (float)(t - R.n_tail); R.denom = (float)t; }
  return R;
}

// The score of one sample: member k's reward at r[k * stride], 2 <= K <= DIAL_MAXENS.  The mean sums in
// member order.  CVaR sorts the K rewards in registers (compile-time indices, +inf padding past K) with
// an odd-even transposition sort: K rounds of adjacent compare-exchanges that swap on a strict `>` only,
// so equal values (ties, -0 / +0) keep member order and the padding never moves.  Then it sums the
// n_tail lowest in ascending order, adds frac * s_{n_tail} as a separate multiply and add, and divides.
// All control flow depends on K and the setting only (uniform across a CTA of the reduction kernel).
// DEV, not HD: the _rn intrinsics are device functions; the emulator build compiles it for the host.
DEV float ens_risk_reduce(const float* r, size_t stride, int K, const EnsRisk& R) {
  if (R.mode == DIAL_ENS_MEAN) {
    float s = r[0];
    for (int k = 1; k < K; ++k) s = __fadd_rn(s, r[(size_t)k * stride]);
    return __fdiv_rn(s, (float)K);
  }
  float s[DIAL_MAXENS];
  bool nan = false;
#pragma unroll
  for (int k = 0; k < DIAL_MAXENS; ++k) {
    s[k] = k < K ? r[(size_t)k * stride] : INFINITY;
    nan = nan || isnan(s[k]);
  }
#pragma unroll
  for (int pass = 0; pass < DIAL_MAXENS; ++pass) {
    if (pass >= K) break;
#pragma unroll
    for (int j = pass & 1; j + 1 < DIAL_MAXENS; j += 2) {
      const float a = s[j], b = s[j + 1];
      const bool swap = a > b;
      s[j] = swap ? b : a;
      s[j + 1] = swap ? a : b;
    }
  }
  float acc = s[0], next = s[1];
#pragma unroll
  for (int j = 1; j < DIAL_MAXENS; ++j) {
    if (j < R.n_tail) acc = __fadd_rn(acc, s[j]);
    if (j == R.n_tail) next = s[j];
  }
  if (R.frac > 0.f) acc = __fadd_rn(acc, __fmul_rn(R.frac, next));
  return nan ? NAN : __fdiv_rn(acc, R.denom);
}

// ---------------------------------------------------------------------------------
// Adapting an ensemble plan to its plant (dial_plan_set_ensemble_adapt): instance b keeps a belief over
// its K members, log-weights L [K] in fp64 and w_k = (float) exp(L_k), updated at every env step from how
// well each member predicted the plant's post-step qvel, and scores samples by the belief-weighted risk
// measure.  ens_belief_kernel and ensemble_reduce_kernel (dial_kernels.cu) run the functions below,
// which the emulator build also runs on the CPU.  DEV, not HD, for the reason given at ens_risk_reduce:
// every operation is a pinned round-to-nearest intrinsic, so that no multiply-add is fused on the GPU.
// ---------------------------------------------------------------------------------
#define DIAL_ENS_LOGLIK_CAP 1.0e4   // C: a member's log-likelihood of one step is at least -C

struct alignas(16) EnsAdapt {
  int32_t on;                 // 0: the instance keeps its belief and scores as without adaptation
  float forget;               // in (0, 1]: L <- forget L + l at every update
  float prune;                // in [0, 1/K): members with w < prune are left out of the score
  int32_t pad_;
  float sigma[DIAL_MAXV];     // the scale of each qvel residual (> 0)
};

// l_k = -min(e_k / 2, C) with e_k = sum_j ((vhat_j - v_j) / sigma_j)^2 in fp64 from the fp32 values, j
// ascending.  A NaN or infinite e_k gives -C.  e_k = 0 gives -0.
DEV double ens_member_loglik(const float* vhat, const float* v, const float* sigma, int nv) {
  double e = 0.0;
  for (int j = 0; j < nv; ++j) {
    const double d = __ddiv_rn(__dsub_rn((double)vhat[j], (double)v[j]), (double)sigma[j]);
    e = __dadd_rn(e, __dmul_rn(d, d));
  }
  const double h = __dmul_rn(e, 0.5);
  return h <= DIAL_ENS_LOGLIK_CAP ? -h : -DIAL_ENS_LOGLIK_CAP;
}

// L_k <- forget L_k + l_k, then L_k <- L_k - (M + log sum_k exp(L_k - M)) with M = max_k L_k, the sum in
// member order; w_k = (float) exp(L_k).  A member at L = -inf stays there with w = 0.
DEV void ens_belief_update(double* L, float* w, const double* ell, int K, double forget) {
  double M = -INFINITY;
  for (int k = 0; k < K; ++k) {
    L[k] = __dadd_rn(__dmul_rn(forget, L[k]), ell[k]);
    M = L[k] > M ? L[k] : M;
  }
  double s = 0.0;
  for (int k = 0; k < K; ++k) s = __dadd_rn(s, exp(__dsub_rn(L[k], M)));
  const double lse = __dadd_rn(M, log(s));
  for (int k = 0; k < K; ++k) {
    L[k] = __dsub_rn(L[k], lse);
    w[k] = (float)exp(L[k]);
  }
}

// The score of one sample under the belief w [K]: member k's reward at r[k * stride].  Member k is kept
// when w_k > 0 and w_k >= prune, or when w_k is the largest weight (so prune < 1/K never empties the
// set); v_k = w_k for the kept members, 0 for the rest, whose rewards are never read into the
// arithmetic.  W = sum_k v_k in member order.  With s_j, v_j the pairs sorted ascending by reward
// (stable in member order, the same transposition sort as ens_risk_reduce):
//   mean:  (sum_k v_k r_k) / W, the sum in member order;
//   worst: the minimum reward of the kept members (the first in member order on ties);
//   CVaR:  tau = alpha W; walking the sorted pairs with v_j > 0 while m < tau: t = min(v_j, tau - m),
//          acc += t s_j, m += t; the score is acc / m: the mean of the worst alpha of the belief's mass.
// Sums start at -0, the exact identity of fp32 addition.  Every operation is fp32 round-to-nearest.  A
// NaN reward of a kept member makes the score NaN.  With uniform weights these equal ens_risk_reduce
// only up to rounding.  Control flow depends on K, the setting and the belief only (uniform per CTA).
DEV float ens_risk_reduce_weighted(const float* r, size_t stride, int K, const EnsRisk& R, const float* w, float prune) {
  float wmax = 0.f;
  for (int k = 0; k < K; ++k) wmax = w[k] > wmax ? w[k] : wmax;
  float s[DIAL_MAXENS], v[DIAL_MAXENS];
  float W = -0.f;
  bool nan = false;
#pragma unroll
  for (int k = 0; k < DIAL_MAXENS; ++k) {
    const float wk = k < K ? w[k] : 0.f;
    const bool kept = wk > 0.f && (wk >= prune || wk == wmax);
    s[k] = kept ? r[(size_t)k * stride] : INFINITY;
    v[k] = kept ? wk : 0.f;
    nan = nan || isnan(s[k]);
    if (kept) W = __fadd_rn(W, wk);
  }
  if (R.mode == DIAL_ENS_MEAN) {
    float acc = -0.f;
#pragma unroll
    for (int k = 0; k < DIAL_MAXENS; ++k)
      if (v[k] > 0.f) acc = __fadd_rn(acc, __fmul_rn(v[k], s[k]));
    return nan ? NAN : __fdiv_rn(acc, W);
  }
  if (R.worst) {
    float m = INFINITY;
#pragma unroll
    for (int k = 0; k < DIAL_MAXENS; ++k)
      if (v[k] > 0.f && s[k] < m) m = s[k];
    return nan ? NAN : m;
  }
#pragma unroll
  for (int pass = 0; pass < DIAL_MAXENS; ++pass) {
    if (pass >= K) break;
#pragma unroll
    for (int j = pass & 1; j + 1 < DIAL_MAXENS; j += 2) {
      const float a = s[j], b = s[j + 1], va = v[j], vb = v[j + 1];
      const bool swap = a > b;
      s[j] = swap ? b : a;
      s[j + 1] = swap ? a : b;
      v[j] = swap ? vb : va;
      v[j + 1] = swap ? va : vb;
    }
  }
  const float tau = __fmul_rn(R.alpha, W);
  float acc = -0.f, m = 0.f;
#pragma unroll
  for (int j = 0; j < DIAL_MAXENS; ++j) {
    if (v[j] > 0.f && m < tau) {
      const float t = fminf(v[j], __fsub_rn(tau, m));
      acc = __fadd_rn(acc, __fmul_rn(t, s[j]));
      m = __fadd_rn(m, t);
    }
  }
  return nan ? NAN : __fdiv_rn(acc, m);
}

// ---------------------------------------------------------------------------------
// Integer structure of the env step as a template policy.  The warp-uniform bounds and selectors the
// env step reads (body / dof / contact counts, tree depth, star chains, pair kind, solver iteration
// counts, physics steps per env step, the reward's environment) come from `SH`:
//   ShapeRT     reads them from the staged model and plan (every model);
//   ShapeFixed  returns the model's structure as compile-time constants (-DDIAL_SHAPE_*: a specialised
//               kernel, built for one model and selected only for plans whose values all match, see
//               shape_matches).  Loops then get constant trip counts and dead branches drop out.
// Lane-varying tables (body depth, joint type, chains, star positions) and every float constant stay
// run-time data: the arithmetic of each row is the same in both kernels, bit for bit.
// ---------------------------------------------------------------------------------
struct ShapeRT {
  static HD int nbody(const DevModel& M) { return M.m.nbody; }
  static HD int nq(const DevModel& M) { return M.m.nq; }
  static HD int nv(const DevModel& M) { return M.m.nv; }
  static HD int nu(const DevModel& M) { return M.m.nu; }
  static HD int maxdepth(const DevModel& M) { return M.maxdepth; }
  static HD int nroot(const DevModel& M) { return M.nroot; }
  static HD int ncon(const DevModel& M) { return M.m.ncon; }
  static HD int nedge(const DevModel& M) { return M.nedge; }
  static HD int nchain(const DevModel& M) { return M.star_nchain; }
  static HD int sb_on(const DevModel& M) { return M.sb_on; }
  static HD int sb_nroot(const DevModel& M) { return M.sb_nroot; }
  static HD int sb_len(const DevModel& M, int l) { return M.sb_len[l]; }
  static HD int pair_kind(const DevModel& M, int k) { return M.m.pair_kind[k]; }
  static HD int iterations(const DevModel& M) { return M.m.iterations; }
  static HD int ls_iterations(const DevModel& M) { return M.m.ls_iterations; }
  static HD int n_frames(const dial_plan_desc& c) { return c.n_frames; }
  static HD int env_id(const dial_plan_desc& c) { return c.env_id; }
  static HD int nfeet(const dial_plan_desc& c) { return c.nfeet; }
};

#ifdef DIAL_SHAPE_NBODY
// Internal linkage: a specialised unit's rollout_kernel<3, 6, ShapeFixed> and shape_matches<ShapeFixed>
// hold its own values and must not be merged with another unit's at link time.  With a fixed contact count
// the compiler split the line search's final `qacc += alpha * search` and `Ma += alpha * mv` updates
// (linesearch_core) into a multiply and an add where the generic kernel fuses them, so rewards differed in
// the last bits on H100; those two updates are written with __fmaf_rn, as the generic kernel compiles them
// (scripts/contraction_diff.py compares the fused/unfused mix of every line in the two kernels).  The fields
// below leave every row bit for bit as the generic kernel computes it.  env_id stays a run-time value
// (inherited from ShapeRT).
namespace {
struct ShapeFixed : ShapeRT {
  static HD constexpr int nbody(const DevModel&) { return DIAL_SHAPE_NBODY; }
  static HD constexpr int nq(const DevModel&) { return DIAL_SHAPE_NQ; }
  static HD constexpr int nv(const DevModel&) { return DIAL_SHAPE_NV; }
  static HD constexpr int nu(const DevModel&) { return DIAL_SHAPE_NU; }
  static HD constexpr int maxdepth(const DevModel&) { return DIAL_SHAPE_MAXDEPTH; }
  static HD constexpr int nroot(const DevModel&) { return DIAL_SHAPE_NROOT; }
  static HD constexpr int nchain(const DevModel&) { return DIAL_SHAPE_NCHAIN; }
  static HD constexpr int sb_on(const DevModel&) { return 1; }
  static HD constexpr int sb_nroot(const DevModel&) { return DIAL_SHAPE_SB_NROOT; }
  static HD constexpr int sb_len(const DevModel&, int) { return DIAL_SHAPE_CHAINLEN; }   // every chain
  static HD constexpr int pair_kind(const DevModel&, int) { return DIAL_SHAPE_PAIR_KIND; }  // every pair
  static HD constexpr int iterations(const DevModel&) { return DIAL_SHAPE_ITERATIONS; }
  static HD constexpr int ls_iterations(const DevModel&) { return DIAL_SHAPE_LS_ITERATIONS; }
  // the library build always defines these; without them (scripts/contraction_diff.py) they stay run-time
#ifdef DIAL_SHAPE_NCON
  static HD constexpr int ncon(const DevModel&) { return DIAL_SHAPE_NCON; }
  static HD constexpr int nedge(const DevModel&) { return DIAL_SHAPE_NEDGE; }
#endif
#ifdef DIAL_SHAPE_NFEET
  static HD constexpr int nfeet(const dial_plan_desc&) { return DIAL_SHAPE_NFEET; }
  static HD constexpr int n_frames(const dial_plan_desc&) { return DIAL_SHAPE_N_FRAMES; }
#endif
};
}  // namespace
#endif

// Whether a kernel compiled for policy SH computes what the run-time kernel computes for this model and
// plan: every value SH fixes equals the model's / plan's own.
template <class SH>
static inline bool shape_matches(const DevModel& M, const dial_plan_desc& c) {
  using R = ShapeRT;
  if (!M.s_on || !R::sb_on(M) || SH::sb_on(M) != R::sb_on(M)) return false;
  if (SH::nbody(M) != R::nbody(M) || SH::nq(M) != R::nq(M) || SH::nv(M) != R::nv(M) || SH::nu(M) != R::nu(M) ||
      SH::maxdepth(M) != R::maxdepth(M) || SH::nroot(M) != R::nroot(M) || SH::ncon(M) != R::ncon(M) ||
      SH::nedge(M) != R::nedge(M) || SH::nchain(M) != R::nchain(M) || SH::sb_nroot(M) != R::sb_nroot(M) ||
      SH::iterations(M) != R::iterations(M) || SH::ls_iterations(M) != R::ls_iterations(M) ||
      SH::n_frames(c) != R::n_frames(c) || SH::env_id(c) != R::env_id(c) || SH::nfeet(c) != R::nfeet(c))
    return false;
  for (int l = 0; l < R::nchain(M); ++l) if (SH::sb_len(M, l) != R::sb_len(M, l)) return false;
  for (int k = 0; k < R::ncon(M); ++k) {
    const int p = M.con_pair[k];
    if (SH::pair_kind(M, p) != R::pair_kind(M, p)) return false;
  }
  return true;
}

// ---------------------------------------------------------------------------------
// small vector / quaternion helpers
// ---------------------------------------------------------------------------------
struct V3 { float x, y, z; };
struct Q4 { float w, x, y, z; };

DEV V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
DEV V3 ld3(const float* p) { return v3(p[0], p[1], p[2]); }
DEV void st3(float* p, V3 a) { p[0] = a.x; p[1] = a.y; p[2] = a.z; }
DEV V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
DEV V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
DEV V3 operator*(V3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }
DEV float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
DEV V3 cross(V3 a, V3 b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
DEV Q4 ldq(const float* p) { Q4 q; q.w = p[0]; q.x = p[1]; q.y = p[2]; q.z = p[3]; return q; }
DEV void stq(float* p, Q4 q) { p[0] = q.w; p[1] = q.x; p[2] = q.y; p[3] = q.z; }
DEV Q4 qmul(Q4 a, Q4 b) {
  Q4 r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x;
  r.z = a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w;
  return r;
}
// MJX math.rotate(vec, quat)
DEV V3 qrot(Q4 q, V3 v) {
  V3 u = v3(q.x, q.y, q.z);
  float s = q.w;
  V3 r = u * (2.f * dot(u, v)) + v * (s * s - dot(u, u));
  return r + cross(u, v) * (2.f * s);
}
DEV Q4 qnormalize(Q4 q) {
  float n = sqrtf(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  float inv = 1.f / (n + 1e-6f * (n == 0.f ? 1.f : 0.f));
  Q4 r; r.w = q.w * inv; r.x = q.x * inv; r.y = q.y * inv; r.z = q.z * inv; return r;
}
DEV void qmat(Q4 q, float* m) {  // row-major 3x3
  float w = q.w, x = q.x, y = q.y, z = q.z;
  m[0] = w * w + x * x - y * y - z * z; m[1] = 2.f * (x * y - w * z); m[2] = 2.f * (x * z + w * y);
  m[3] = 2.f * (x * y + w * z); m[4] = w * w - x * x + y * y - z * z; m[5] = 2.f * (y * z - w * x);
  m[6] = 2.f * (x * z - w * y); m[7] = 2.f * (y * z + w * x); m[8] = w * w - x * x - y * y + z * z;
}
DEV Q4 axisangle(V3 axis, float angle) {
  float s, c;
  fast_sincos(0.5f * angle, s, c);   // |angle/2| < pi: SFU sin/cos (abs err ~4e-7), same code in every instantiation
  Q4 q; q.w = c; q.x = axis.x * s; q.y = axis.y * s; q.z = axis.z * s; return q;
}

// 128 / 64-bit shared-memory accesses (addresses must be 16 / 8-byte aligned)
struct F4 { float x, y, z, w; };
DEV F4 ld4(const float* p) {
#ifdef DIAL_HOST_EMUL
  F4 r; r.x = p[0]; r.y = p[1]; r.z = p[2]; r.w = p[3]; return r;
#else
  const float4 v = *reinterpret_cast<const float4*>(p);
  F4 r; r.x = v.x; r.y = v.y; r.z = v.z; r.w = v.w; return r;
#endif
}
DEV void st4(float* p, float a, float b, float c, float d) {
#ifdef DIAL_HOST_EMUL
  p[0] = a; p[1] = b; p[2] = c; p[3] = d;
#else
  *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
#endif
}
DEV void ld2(const float* p, float& a, float& b) {
#ifdef DIAL_HOST_EMUL
  a = p[0]; b = p[1];
#else
  const float2 v = *reinterpret_cast<const float2*>(p);
  a = v.x; b = v.y;
#endif
}
DEV void st2(float* p, float a, float b) {
#ifdef DIAL_HOST_EMUL
  p[0] = a; p[1] = b;
#else
  *reinterpret_cast<float2*>(p) = make_float2(a, b);
#endif
}
// spatial vectors in the slab: cdof / cdofdot rows are padded to CDS = 8 floats, cinert / crb rows to
// CIS = 12, so that a row is one 128-bit + one 64-bit access (two + one for the inertias)
#define CDS 8
#define CIS 12
DEV void ld6(const float* p, float* o) {
  F4 a = ld4(p);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
  ld2(p + 4, o[4], o[5]);
}
DEV void st6(float* p, const float* v) {
  st4(p, v[0], v[1], v[2], v[3]);
  st2(p + 4, v[4], v[5]);
}
DEV void ld10(const float* p, float* o) {
  F4 a = ld4(p), b = ld4(p + 4);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
  ld2(p + 8, o[8], o[9]);
}

// spatial helpers on [ang(3), lin(3)] vectors
DEV void mcross(const float* u, const float* v, float* r) {  // motion cross
  V3 ua = ld3(u), ul = ld3(u + 3), va = ld3(v), vl = ld3(v + 3);
  st3(r, cross(ua, va));
  st3(r + 3, cross(ul, va) + cross(ua, vl));
}
DEV void mcross_force(const float* v, const float* f, float* r) {
  V3 va = ld3(v), vl = ld3(v + 3), fa = ld3(f), fl = ld3(f + 3);
  st3(r, cross(va, fa) + cross(vl, fl));
  st3(r + 3, cross(va, fl));
}
// cinert (10: Ixx Iyy Izz Ixy Ixz Iyz | m*off | m) times motion vector
DEV void inert_mul(const float* ci, const float* v, float* r) {
  V3 va = ld3(v), vl = ld3(v + 3), pos = ld3(ci + 6);
  float m = ci[9];
  V3 ang = v3(ci[0] * va.x + ci[3] * va.y + ci[4] * va.z,
              ci[3] * va.x + ci[1] * va.y + ci[5] * va.z,
              ci[4] * va.x + ci[5] * va.y + ci[2] * va.z) + cross(pos, vl);
  V3 vel = vl * m - cross(pos, va);
  st3(r, ang); st3(r + 3, vel);
}
DEV float dot6(const float* a, const float* b) {
  return (a[0] * b[0] + a[1] * b[1] + a[2] * b[2]) + (a[3] * b[3] + a[4] * b[4] + a[5] * b[5]);
}

DEV float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += shfl_xor(v, o);
  return v;
}
DEV void warp_sum3(float& a, float& b, float& c) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { a += shfl_xor(a, o); b += shfl_xor(b, o); c += shfl_xor(c, o); }
}

// ---------------------------------------------------------------------------------
// Threefry-2x32 (20 rounds) and the JAX legacy normal sampler
// (jax.random.normal at core/dial_core.py:107-109; third party, restated)
// ---------------------------------------------------------------------------------
HD uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
HD void threefry2x32(uint32_t k0, uint32_t k1, uint32_t& x0, uint32_t& x1) {
  uint32_t ks2 = k0 ^ k1 ^ 0x1BD11BDAu;
  x0 += k0; x1 += k1;
#define TF_R(r) { x0 += x1; x1 = rotl32(x1, r); x1 ^= x0; }
  TF_R(13) TF_R(15) TF_R(26) TF_R(6)   x0 += k1;  x1 += ks2 + 1u;
  TF_R(17) TF_R(29) TF_R(16) TF_R(24)  x0 += ks2; x1 += k0 + 2u;
  TF_R(13) TF_R(15) TF_R(26) TF_R(6)   x0 += k0;  x1 += k1 + 3u;
  TF_R(17) TF_R(29) TF_R(16) TF_R(24)  x0 += k1;  x1 += ks2 + 4u;
  TF_R(13) TF_R(15) TF_R(26) TF_R(6)   x0 += ks2; x1 += k0 + 5u;
#undef TF_R
}
// rng, key = jax.random.split(rng) (legacy layout: counters [0,1,2,3] -> halves (0,1) | (2,3)):
// the sampling key (second half); split_rng gives the first half (the new rng)
HD void split_key(uint32_t k0, uint32_t k1, uint32_t& key0, uint32_t& key1) {
  uint32_t a0 = 0, b0 = 2, a1 = 1, b1 = 3;
  threefry2x32(k0, k1, a0, b0);
  threefry2x32(k0, k1, a1, b1);
  key0 = b0; key1 = b1;
}
HD void split_rng(uint32_t k0, uint32_t k1, uint32_t& r0, uint32_t& r1) {
  uint32_t a0 = 0, b0 = 2, a1 = 1, b1 = 3;
  threefry2x32(k0, k1, a0, b0);
  threefry2x32(k0, k1, a1, b1);
  r0 = a0; r1 = a1;
}
// element `i` of jax.random.bits(key, (n,)) with threefry_partitionable=False
DEV uint32_t jax_bits_legacy(uint32_t k0, uint32_t k1, uint32_t i, uint32_t n) {
  uint32_t half = (n + 1u) >> 1;
  uint32_t x0, x1;
  if (i < half) { x0 = i; x1 = i + half; } else { x0 = i - half; x1 = i; }
  bool second = i >= half;
  if (x1 >= n) x1 = 0u;  // odd n: the counter array is padded with one zero
  threefry2x32(k0, k1, x0, x1);
  return second ? x1 : x0;
}
// XLA's single-precision erfinv (Giles' polynomials)
DEV float erfinv_f32(float x) {
  float w = -log1pf(-x * x);
  float p;
  if (w < 5.f) {
    w -= 2.5f;
    p = 2.81022636e-08f;
    p = 3.43273939e-07f + p * w; p = -3.5233877e-06f + p * w; p = -4.39150654e-06f + p * w;
    p = 0.00021858087f + p * w; p = -0.00125372503f + p * w; p = -0.00417768164f + p * w;
    p = 0.246640727f + p * w; p = 1.50140941f + p * w;
  } else {
    w = sqrtf(w) - 3.f;
    p = -0.000200214257f;
    p = 0.000100950558f + p * w; p = 0.00134934322f + p * w; p = -0.00367342844f + p * w;
    p = 0.00573950773f + p * w; p = -0.0076224613f + p * w; p = 0.00943887047f + p * w;
    p = 1.00167406f + p * w; p = 2.83297682f + p * w;
  }
  return p * x;
}
DEV float jax_normal_legacy(uint32_t k0, uint32_t k1, uint32_t i, uint32_t n) {
  uint32_t bits = jax_bits_legacy(k0, k1, i, n);
  float f = __uint_as_float((bits >> 9) | 0x3F800000u) - 1.0f;
  const float lo = -0.99999994f;  // nextafter(-1, 0)
  float u = fmaxf(lo, f * 2.0f + lo);
  return 1.41421356237f * erfinv_f32(u);
}

// ---------------------------------------------------------------------------------
// per-instance observation (dial_plan_set_instance_observation)
// ---------------------------------------------------------------------------------
// Instance b's observation setting (dial_plan_set_instance_observation): the observation delay k in control
// steps, whether the instance observes (k > 0 or some sigma > 0; else it plans from its plant state), the key
// a reset restarts its noise from, and the noise standard deviations: sigma[i] on qpos dof i (tangent space),
// sigma[nv + i] on qvel dof i.
struct alignas(8) ObsSetting {
  int32_t k;
  int32_t on;
  uint32_t key[2];
  float sigma[2 * DIAL_MAXV];
};
#define DIAL_OBSRING (DIAL_MAXDELAY + 1)   // plant records of one instance: ages 0..DIAL_MAXDELAY
// An instance's ring of plant records: the slot of the newest, the records since the reset (counting the
// seed, saturating at DIAL_OBSRING; 0: the next observe step seeds), the running noise key and the key of
// the last draw.
struct alignas(8) ObsRing {
  int32_t head, count;
  uint32_t key[2], sub[2];
};
// One instance's slices of the buffers an observe step reads and writes: the plant state and the action its
// last env step applied (null: none), the ring's records [DIAL_OBSRING][*], the observation, the planning
// state the prediction starts from, the prediction's actions [DIAL_MAXDELAY][nu] and the pending actions of
// the delay queue [DIAL_MAXDELAY][nu] (null: no queue).
struct ObsView {
  const float *qpos, *qvel, *warm, *act;
  const int32_t* cnt;
  float *rq, *rv, *rw, *ra;
  int32_t* rc;
  float *oq, *ov, *ow;
  int32_t* oc;
  float *pq, *pv, *pw;
  int32_t* pc;
  float* seq;
  const float* pending;
};
// The ring after one observe step: an observing instance pushes a record in a step with an env step, and
// seeds one after a reset; each new record draws its noise key, (key, sub) = split(key).
DEV bool observe_pushes(const ObsSetting& s, const ObsRing& r, bool env_step) { return s.on && (r.count == 0 || env_step); }
DEV ObsRing observe_advance(const ObsSetting& s, ObsRing r, bool env_step) {
  if (!observe_pushes(s, r, env_step)) return r;
  r.head = r.count == 0 ? 0 : (r.head + 1 == DIAL_OBSRING ? 0 : r.head + 1);
  r.count = r.count < DIAL_OBSRING ? r.count + 1 : DIAL_OBSRING;
  uint32_t n0, n1, s0, s1;
  split_rng(r.key[0], r.key[1], n0, n1);
  split_key(r.key[0], r.key[1], s0, s1);
  r.key[0] = n0; r.key[1] = n1; r.sub[0] = s0; r.sub[1] = s1;
  return r;
}
// The age of the record an instance observes: min(k, count - 1), the oldest record while the ring fills.
DEV int observe_age(const ObsSetting& s, const ObsRing& r) {
  if (!s.on) return 0;
  return s.k < r.count - 1 ? s.k : r.count - 1;
}
// Stage 1 of an observe step, for the elements a = a0, a0 + da, ... (a CTA passes its threads): when the step
// pushes (observe_pushes), the new record (slot r1.head, r1 = observe_advance(...)) takes the plant state, its
// counters and the applied action (zero without one).  Each element is read and written by one caller only.
DEV void observe_record(bool push, const ObsRing& r1, const ObsView& V, int nq, int nv, int nu, int a0, int da) {
  if (!push) return;
  const int h = r1.head;
  for (int i = a0; i < nq; i += da) V.rq[h * nq + i] = V.qpos[i];
  for (int i = a0; i < nv; i += da) { V.rv[h * nv + i] = V.qvel[i]; V.rw[h * nv + i] = V.warm[i]; }
  for (int i = a0; i < nu; i += da) V.ra[h * nu + i] = V.act ? V.act[i] : 0.f;
  if (a0 == 0) { V.rc[2 * h] = V.cnt[0]; V.rc[2 * h + 1] = V.cnt[1]; }
}
// x + sigma eps, and x itself, bit for bit, where sigma is 0
DEV float observe_noisy(float x, float sigma, float eps) { return sigma == 0.f ? x : fmaf(sigma, eps, x); }
// q composed with the rotation w (body frame) as physics_step integrates a free joint's orientation:
// qnormalize(q * axisangle(w / |w|, |w|))
DEV Q4 observe_rotate(Q4 q, V3 w) {
  const float nrm = sqrtf(dot(w, w));
  const V3 ax = w * (1.f / (nrm + 1e-6f * (nrm == 0.f ? 1.f : 0.f)));
  return qnormalize(qmul(q, axisangle(ax, nrm)));
}
// Stage 2 of an observe step (after stage 1 of every element), for the elements a0, a0 + da, ...: the
// observation (the record `age` pushes back plus the noise of the newest record's draw; the plant state of an
// instance that does not observe) into V.o* and V.p*, and the prediction's actions: `age` history rows (the
// actions applied since the observed record, oldest first), then the d pending rows, then zero rows.  The
// prediction length is age + d (the caller applies the predict flag).
DEV void observe_emit(const ObsSetting& s, const ObsRing& r1, const dial_model_desc& m, int d, const ObsView& V,
                      int a0, int da) {
  const int nq = m.nq, nv = m.nv, nu = m.nu;
  const int age = observe_age(s, r1);
  const int h = s.on ? (r1.head - age < 0 ? r1.head - age + DIAL_OBSRING : r1.head - age) : 0;
  const float* q = s.on ? V.rq + h * nq : V.qpos;
  const float* v = s.on ? V.rv + h * nv : V.qvel;
  const float* w = s.on ? V.rw + h * nv : V.warm;
  const int32_t* c = s.on ? V.rc + 2 * h : V.cnt;
  const uint32_t k0 = r1.sub[0], k1 = r1.sub[1];
  const uint32_t n = 2u * (uint32_t)nv;
  const float* sg = s.sigma;
  for (int j = a0; j < m.njnt; j += da) {
    const int qa = m.jnt_qposadr[j], dd = m.jnt_dofadr[j], t = m.jnt_type[j];
    int qr = -1, dr = -1;   // quaternion address and its three rotation dofs (free and ball joints)
    if (t == JNT_FREE) {
      for (int i = 0; i < 3; ++i) {
        const float x = !s.on ? q[qa + i] : observe_noisy(q[qa + i], sg[dd + i],
                                                          sg[dd + i] == 0.f ? 0.f : jax_normal_legacy(k0, k1, dd + i, n));
        V.oq[qa + i] = x; V.pq[qa + i] = x;
      }
      qr = qa + 3; dr = dd + 3;
    } else if (t == JNT_BALL) {
      qr = qa; dr = dd;
    } else {
      const float x = !s.on || sg[dd] == 0.f ? q[qa] : observe_noisy(q[qa], sg[dd], jax_normal_legacy(k0, k1, dd, n));
      V.oq[qa] = x; V.pq[qa] = x;
    }
    if (qr >= 0) {
      Q4 o = ldq(q + qr);
      if (s.on && (sg[dr] != 0.f || sg[dr + 1] != 0.f || sg[dr + 2] != 0.f)) {
        V3 e = v3(0.f, 0.f, 0.f);
        if (sg[dr] != 0.f) e.x = sg[dr] * jax_normal_legacy(k0, k1, dr, n);
        if (sg[dr + 1] != 0.f) e.y = sg[dr + 1] * jax_normal_legacy(k0, k1, dr + 1, n);
        if (sg[dr + 2] != 0.f) e.z = sg[dr + 2] * jax_normal_legacy(k0, k1, dr + 2, n);
        o = observe_rotate(o, e);
      }
      stq(V.oq + qr, o); stq(V.pq + qr, o);
    }
  }
  for (int i = a0; i < nv; i += da) {
    const float x = !s.on || sg[nv + i] == 0.f ? v[i] : observe_noisy(v[i], sg[nv + i], jax_normal_legacy(k0, k1, nv + i, n));
    V.ov[i] = x; V.pv[i] = x;
    V.ow[i] = w[i]; V.pw[i] = w[i];
  }
  if (a0 == 0) { V.oc[0] = c[0]; V.oc[1] = c[1]; V.pc[0] = c[0]; V.pc[1] = c[1]; }
  for (int a = a0; a < nu; a += da)
    for (int j = 0; j < DIAL_MAXDELAY; ++j) {
      float u = 0.f;
      if (j < age) {
        const int back = age - 1 - j, sl = r1.head - back;   // the record j + 1 steps after the observed one
        u = V.ra[(sl < 0 ? sl + DIAL_OBSRING : sl) * nu + a];
      } else if (j < age + d && V.pending) {
        u = V.pending[(j - age) * nu + a];
      }
      V.seq[j * nu + a] = u;
    }
}

// ---------------------------------------------------------------------------------
// per-instance pushes (dial_plan_set_instance_pushes)
// ---------------------------------------------------------------------------------
// This is a separate, plain fp64 restatement of the kinematics, the COM-frame inertias and motion axes and the
// CRB mass matrix, not a reuse of physics_step's sections: those are fused and tuned for the rollout kernel's
// instruction stream, and sharing them would put this feature into rollout_kernel.  It runs only in an env step
// at which some push fires, on one warp per instance (push_kernel), so its cost does not matter.
//
// Instance b's push table: its n entries (dial_push, include/dial_b200.h).
struct alignas(16) PushTable {
  int32_t n;
  int32_t pad[3];
  dial_push e[DIAL_MAXPUSH];
};
// entry e fires after the env step whose post-step counter is `step`: step in [e.step, e.step + n_steps)
HD bool push_fires(const dial_push& e, int step) { return step >= e.step && step - e.step < e.n_steps; }
HD bool push_any(const PushTable& T, int step) {
  for (int i = 0; i < T.n; ++i)
    if (push_fires(T.e[i], step)) return true;
  return false;
}
// The fp64 workspace of one instance's push (shared memory in push_kernel): the body frames, the subtree COM of
// each body's tree root, the composite inertias (cinert layout, COM frame), the dofs' motion axes, the mass
// matrix (its Cholesky factor after push_solve) and the generalized impulse (Delta qvel after push_solve).
struct PushWork {
  double xpos[DIAL_MAXB][3], xquat[DIAL_MAXB][4], xmat[DIAL_MAXB][9];
  double xipos[DIAL_MAXB][3], ximat[DIAL_MAXB][9];
  double xanchor[DIAL_MAXB][3], xaxis[DIAL_MAXB][3];
  double com[DIAL_MAXB][3];
  double crb[DIAL_MAXB][10];
  double cdof[DIAL_MAXV][6];
  double M[DIAL_MAXV][DIAL_MAXV];
  double g[DIAL_MAXV];
};
HD void pd_qmul(const double* a, const double* b, double* r) {
  const double w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  const double x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  const double y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  const double z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
HD void pd_qrot(const double* q, const double* v, double* r) {   // mjx math.rotate
  const double s = q[0], uv = q[1] * v[0] + q[2] * v[1] + q[3] * v[2], uu = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  const double c[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  for (int i = 0; i < 3; ++i) r[i] = 2.0 * uv * q[1 + i] + (s * s - uu) * v[i] + 2.0 * s * c[i];
}
HD void pd_qnormalize(double* q) {
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double d = n + (n == 0.0 ? 1e-6 : 0.0);
  for (int i = 0; i < 4; ++i) q[i] /= d;
}
HD void pd_qmat(const double* q, double* m) {   // row-major 3x3
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  m[0] = w * w + x * x - y * y - z * z; m[1] = 2 * (x * y - w * z); m[2] = 2 * (x * z + w * y);
  m[3] = 2 * (x * y + w * z); m[4] = w * w - x * x + y * y - z * z; m[5] = 2 * (y * z - w * x);
  m[6] = 2 * (x * z - w * y); m[7] = 2 * (y * z + w * x); m[8] = w * w - x * x - y * y + z * z;
}
HD void pd_cross(const double* a, const double* b, double* r) {
  const double x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
// cinert (10) times a motion vector (6) (mjx inert_mul)
HD void pd_inert_mul(const double* ci, const double* v, double* r) {
  const double I[9] = {ci[0], ci[3], ci[4], ci[3], ci[1], ci[5], ci[4], ci[5], ci[2]};
  double pw[3], pv[3];
  pd_cross(ci + 6, v + 3, pw);
  pd_cross(ci + 6, v, pv);
  for (int i = 0; i < 3; ++i) {
    r[i] = I[3 * i] * v[0] + I[3 * i + 1] * v[1] + I[3 * i + 2] * v[2] + pw[i];
    r[3 + i] = ci[9] * v[3 + i] - pv[i];
  }
}
// Stage 1 of a push (one caller): the body frames at qpos (quaternions normalised as mjx.kinematics does), the
// subtree COM of every tree root, each body's inertia about its root's COM, the composite inertias (each body's
// summed over its subtree, the world's zero) and the dofs' motion axes about their root's COM, on the model m
// (free, hinge and slide joints).
DEV void push_kinematics(const dial_model_desc& m, const float* qpos, PushWork& W) {
  const int nb = m.nbody;
  for (int i = 0; i < 3; ++i) { W.xpos[0][i] = 0.0; W.xanchor[0][i] = 0.0; W.xaxis[0][i] = 0.0; }
  W.xquat[0][0] = 1.0; W.xquat[0][1] = 0.0; W.xquat[0][2] = 0.0; W.xquat[0][3] = 0.0;
  for (int b = 1; b < nb; ++b) {
    const int p = m.body_parentid[b];
    double bp[3], bq[4], pos[3], quat[4];
    for (int i = 0; i < 3; ++i) bp[i] = m.body_pos[b][i];
    for (int i = 0; i < 4; ++i) bq[i] = m.body_quat[b][i];
    pd_qrot(W.xquat[p], bp, pos);
    for (int i = 0; i < 3; ++i) pos[i] += W.xpos[p][i];
    pd_qmul(W.xquat[p], bq, quat);
    double anchor[3] = {0.0, 0.0, 0.0}, axis[3] = {0.0, 0.0, 0.0};
    const int j = m.body_jntadr[b];
    if (j >= 0) {
      const int qa = m.jnt_qposadr[j], t = m.jnt_type[j];
      if (t == JNT_FREE) {
        for (int i = 0; i < 3; ++i) { pos[i] = qpos[qa + i]; anchor[i] = pos[i]; }
        axis[2] = 1.0;
        for (int i = 0; i < 4; ++i) quat[i] = qpos[qa + 3 + i];
        pd_qnormalize(quat);
      } else {
        double jp[3], ja[3], r[3];
        for (int i = 0; i < 3; ++i) { jp[i] = m.jnt_pos[j][i]; ja[i] = m.jnt_axis[j][i]; }
        pd_qrot(quat, jp, r);
        for (int i = 0; i < 3; ++i) anchor[i] = r[i] + pos[i];
        pd_qrot(quat, ja, axis);
        const double ang = (double)qpos[qa] - (double)m.qpos0[qa];
        if (t == JNT_HINGE) {
          const double s = sin(0.5 * ang), c = cos(0.5 * ang);
          const double ql[4] = {c, ja[0] * s, ja[1] * s, ja[2] * s};
          double q2[4];
          pd_qmul(quat, ql, q2);
          for (int i = 0; i < 4; ++i) quat[i] = q2[i];
          pd_qrot(quat, jp, r);
          for (int i = 0; i < 3; ++i) pos[i] = anchor[i] - r[i];
        } else {   // slide
          for (int i = 0; i < 3; ++i) pos[i] += axis[i] * ang;
        }
      }
    }
    pd_qnormalize(quat);
    for (int i = 0; i < 3; ++i) { W.xpos[b][i] = pos[i]; W.xanchor[b][i] = anchor[i]; W.xaxis[b][i] = axis[i]; }
    for (int i = 0; i < 4; ++i) W.xquat[b][i] = quat[i];
  }
  // inertial frames; the mass-weighted sums of each tree root (accumulated in com, normalised below)
  double msum[DIAL_MAXB];
  for (int b = 0; b < nb; ++b) {
    double ip[3], iq[4], q2[4], r[3];
    for (int i = 0; i < 3; ++i) ip[i] = m.body_ipos[b][i];
    for (int i = 0; i < 4; ++i) iq[i] = m.body_iquat[b][i];
    pd_qmat(W.xquat[b], W.xmat[b]);
    pd_qrot(W.xquat[b], ip, r);
    for (int i = 0; i < 3; ++i) W.xipos[b][i] = W.xpos[b][i] + r[i];
    pd_qmul(W.xquat[b], iq, q2);
    pd_qmat(q2, W.ximat[b]);
    msum[b] = 0.0;
    for (int i = 0; i < 3; ++i) W.com[b][i] = 0.0;
  }
  for (int b = 0; b < nb; ++b) {
    const int r = m.body_rootid[b];
    msum[r] += (double)m.body_mass[b];
    for (int i = 0; i < 3; ++i) W.com[r][i] += (double)m.body_mass[b] * W.xipos[b][i];
  }
  for (int b = 0; b < nb; ++b) {   // roots first: a root is its own root and precedes its subtree
    const int r = m.body_rootid[b];
    if (r != b) continue;
    for (int i = 0; i < 3; ++i) W.com[b][i] = msum[b] < (double)DIAL_MINVAL ? W.xipos[b][i] : W.com[b][i] / msum[b];
  }
  for (int b = 0; b < nb; ++b) {
    const int r = m.body_rootid[b];
    if (r != b) for (int i = 0; i < 3; ++i) W.com[b][i] = W.com[r][i];
  }
  // cinert of each body about its root's COM: R diag(I) R^T + m (|o|^2 1 - o o^T), [Ixx Iyy Izz Ixy Ixz Iyz | m o | m]
  for (int b = 0; b < nb; ++b) {
    const double mass = m.body_mass[b];
    double o[3], I[9];
    for (int i = 0; i < 3; ++i) o[i] = W.xipos[b][i] - W.com[b][i];
    const double o2 = o[0] * o[0] + o[1] * o[1] + o[2] * o[2];
    for (int i = 0; i < 3; ++i)
      for (int k = 0; k < 3; ++k) {
        double s = 0.0;
        for (int l = 0; l < 3; ++l) s += W.ximat[b][3 * i + l] * (double)m.body_inertia[b][l] * W.ximat[b][3 * k + l];
        I[3 * i + k] = s + mass * ((i == k ? o2 : 0.0) - o[i] * o[k]);
      }
    double* c = W.crb[b];
    c[0] = I[0]; c[1] = I[4]; c[2] = I[8]; c[3] = I[1]; c[4] = I[2]; c[5] = I[5];
    for (int i = 0; i < 3; ++i) c[6 + i] = o[i] * mass;
    c[9] = mass;
  }
  for (int b = nb - 1; b > 0; --b) {
    const int p = m.body_parentid[b];
    if (p > 0) for (int i = 0; i < 10; ++i) W.crb[p][i] += W.crb[b][i];
  }
  for (int i = 0; i < 10; ++i) W.crb[0][i] = 0.0;
  // the motion axes of the dofs about their root's COM: [angular | linear]
  for (int b = 1; b < nb; ++b) {
    const int j = m.body_jntadr[b];
    if (j < 0) continue;
    const int d = m.jnt_dofadr[j], t = m.jnt_type[j];
    double off[3];
    for (int i = 0; i < 3; ++i) off[i] = W.com[b][i] - W.xanchor[b][i];
    if (t == JNT_FREE) {
      for (int i = 0; i < 3; ++i) {
        double* tr = W.cdof[d + i];
        double* rot = W.cdof[d + 3 + i];
        for (int k = 0; k < 6; ++k) tr[k] = 0.0;
        tr[3 + i] = 1.0;
        const double ax[3] = {W.xmat[b][i], W.xmat[b][3 + i], W.xmat[b][6 + i]};
        for (int k = 0; k < 3; ++k) rot[k] = ax[k];
        pd_cross(ax, off, rot + 3);
      }
    } else if (t == JNT_HINGE) {
      for (int k = 0; k < 3; ++k) W.cdof[d][k] = W.xaxis[b][k];
      pd_cross(W.xaxis[b], off, W.cdof[d] + 3);
    } else {
      for (int k = 0; k < 3; ++k) { W.cdof[d][k] = 0.0; W.cdof[d][3 + k] = W.xaxis[b][k]; }
    }
  }
}
// Stage 2 of a push (after stage 1), for the dofs i = a0, a0 + da, ... < nv (a warp passes its lanes): row i of
// the CRB mass matrix M = cdof^T crb cdof on the ancestor pattern, armature on the diagonal, and the generalized
// impulse g[i] = sum over the entries firing at `step` of cdof_i . [torque + (p - c) x force; force] dt, p the
// entry's world point and c its body's root COM (J^T [torque; force] dt).  Each caller writes its own rows only.
DEV void push_rows(const DevModel& D, const PushTable& T, int step, double dt, PushWork& W, int a0, int da) {
  const dial_model_desc& m = D.m;
  const int nv = m.nv;
  for (int i = a0; i < nv; i += da) {
    double vi[6];
    pd_inert_mul(W.crb[m.dof_bodyid[i]], W.cdof[i], vi);
    for (int j = 0; j < nv; ++j) {
      double s = 0.0;
      if ((D.dof_ancmask[i] >> j) & 1u) {
        for (int k = 0; k < 6; ++k) s += vi[k] * W.cdof[j][k];
      } else if ((D.dof_ancmask[j] >> i) & 1u) {
        double vj[6];
        pd_inert_mul(W.crb[m.dof_bodyid[j]], W.cdof[j], vj);
        for (int k = 0; k < 6; ++k) s += vj[k] * W.cdof[i][k];
      }
      W.M[i][j] = s + (i == j ? (double)m.dof_armature[i] : 0.0);
    }
    double g = 0.0;
    for (int e = 0; e < T.n; ++e) {
      const dial_push& P = T.e[e];
      if (!push_fires(P, step) || !((D.body_dofmask[P.body] >> i) & 1u)) continue;
      double pw[3], f[3], tq[3];
      for (int k = 0; k < 3; ++k) {
        pw[k] = W.xpos[P.body][k] + W.xmat[P.body][3 * k] * (double)P.pos[0] + W.xmat[P.body][3 * k + 1] * (double)P.pos[1] +
                W.xmat[P.body][3 * k + 2] * (double)P.pos[2] - W.com[P.body][k];
        f[k] = P.force[k];
      }
      pd_cross(pw, f, tq);
      for (int k = 0; k < 3; ++k) g += W.cdof[i][k] * ((double)P.torque[k] + tq[k]) + W.cdof[i][3 + k] * f[k];
    }
    W.g[i] = g * dt;
  }
}
// Stage 3 of a push (one caller, after stage 2 of every row): g = M^-1 g by a dense Cholesky factorisation
// M = L L^T in place (the lower triangle) and two triangular solves.
DEV void push_solve(int nv, PushWork& W) {
  for (int k = 0; k < nv; ++k) {
    double d = W.M[k][k];
    for (int l = 0; l < k; ++l) d -= W.M[k][l] * W.M[k][l];
    d = sqrt(d);
    W.M[k][k] = d;
    for (int i = k + 1; i < nv; ++i) {
      double s = W.M[i][k];
      for (int l = 0; l < k; ++l) s -= W.M[i][l] * W.M[k][l];
      W.M[i][k] = s / d;
    }
  }
  for (int i = 0; i < nv; ++i) {
    double s = W.g[i];
    for (int l = 0; l < i; ++l) s -= W.M[i][l] * W.g[l];
    W.g[i] = s / W.M[i][i];
  }
  for (int i = nv - 1; i >= 0; --i) {
    double s = W.g[i];
    for (int l = i + 1; l < nv; ++l) s -= W.M[l][i] * W.g[l];
    W.g[i] = s / W.M[i][i];
  }
}
// qvel + Delta qvel, rounded once; a zero Delta leaves qvel bit for bit
HD float push_add(float v, double dv) { return dv == 0.0 ? v : (float)((double)v + dv); }

// ---------------------------------------------------------------------------------
// per-warp context
// ---------------------------------------------------------------------------------
// "Compact chain coordinates": the mass matrix M and the Newton Hessian H = M + J^T D J of
// a kinematic tree are non-zero only at (i, j) with j an ancestor-or-self dof of i.  Row i is
// therefore stored as R[c] = H[i][chain_i[c]], c = 0..n_i-1, where chain_i = (i, parent(i),
// ..., root dof) — and because the chain of an ancestor is a suffix of the chain of its
// descendants, every tree operation below (reverse-order Cholesky L^T L without fill-in,
// triangular solves, J^T D J rank-1 updates, M x) becomes index-free: an ancestor `a` of
// pivot `k` sits at position n_k - n_a of k's row and needs positions n_k - n_a + c.
struct WarpCtx {
  const DevModel* M;   // in shared memory
  const DevPlan* P;    // in shared memory
  float* s;            // this warp's slab
  int lane;
  int nch;             // chain length of this lane's dof (0: lane is not a dof)
  int ndesc;           // descendant dofs (they follow the dof contiguously, DFS order)
  int mylevel;         // elimination level of the dof (leaves = 0), -1 for non-dof lanes
  int parent;          // parent dof or -1
  int midsync;         // lock-step CTAs: extra CTA barrier before the Newton loop
  int itersync;        // lock-step level 3 (dense path): CTA barrier per Newton iteration
  float* dbg;          // optional counters (tests / tuning): [0] physics steps, [1] Newton iterations
  int chain[DIAL_MAXCHAIN];
  // star layout constants of this lane (star variants; DevModel::s_*)
  int s_pos;           // star position of this lane's dof (0 for non-dof lanes)
  int s_col;           // its column inside a row: root index a, or NRP + depth for a chain dof
  int s_cb;            // first position of its chain (NRP for root / non-dof lanes)
  int s_chain;         // chain id, -1: root dof, -2: not a dof
  int s_depth;         // depth inside the chain / root index
  int s_top;           // first dof of its chain
  uint32_t s_conmask;  // contacts whose rows can be non-zero in this lane's column
  int e_cb;            // edge lanes: first position of the contact's chain (NRP if the body hangs off the root chain)
#ifdef DIAL_TERRAIN
  const DevTerrain* ter;   // this row's terrain, null on the flat floor
#endif
};

#define SM(name) (w.s + w.M->o_##name)
#define MC DIAL_MAXCHAIN

// H = L^T L (reverse order, no fill-in).  R: this lane's compact row, overwritten by the
// factor row (diagonal = sqrt pivot); *invd = 1/L[i][i].  Factor rows are published in
// SM(L) for the solves.  One syncwarp per elimination level.
DEV void factor_LTL(WarpCtx& w, float* R, float& invd) {
  const DevModel& M = *w.M;
  float* Lb = SM(L);
  const int lane = w.lane;
  for (int lv = 0; lv < M.nlevel; ++lv) {
    if (w.mylevel == lv) {
      float inv = rsqrtf(fmaxf(R[0], DIAL_MINVAL));
      invd = inv;
      R[0] = R[0] * inv;
#pragma unroll
      for (int c = 1; c < MC; ++c) R[c] *= inv;
#pragma unroll
      for (int c = 0; c < MC; ++c)
        if (c < w.nch) Lb[lane * MC + c] = R[c];
    }
    syncwarp();
    if (w.mylevel > lv) {
      for (int pi = M.level_adr[lv]; pi < M.level_adr[lv + 1]; ++pi) {
        const int k = M.level_dofs[pi];
        if ((M.dof_ancmask[k] >> lane) & 1u) {
          const float* Lk = Lb + k * MC + (M.dof_nchain[k] - w.nch);
          const float l0 = Lk[0];
#pragma unroll
          for (int c = 0; c < MC; ++c)
            if (c < w.nch) R[c] -= l0 * Lk[c];
        }
      }
    }
  }
}

// solve (L^T L) x = g.  Lane d holds g_d / returns x_d; R, invd from factor_LTL.
DEV float solve_LTL(WarpCtx& w, const float* R, float invd, float g) {
  const DevModel& M = *w.M;
  const float* Lb = SM(L);
  float* vec = SM(vec);
  float* xch = SM(xch);  // published ancestor chains of x: xch[d][c] = x[chain_d[c]]
  const int lane = w.lane;
  float y = g;
  // L^T y = g : leaves -> root
  for (int lv = 0; lv < M.nlevel; ++lv) {
    if (w.mylevel == lv) { y *= invd; vec[lane] = y; }
    syncwarp();
    if (w.mylevel > lv) {
      for (int pi = M.level_adr[lv]; pi < M.level_adr[lv + 1]; ++pi) {
        const int k = M.level_dofs[pi];
        if ((M.dof_ancmask[k] >> lane) & 1u) y -= Lb[k * MC + (M.dof_nchain[k] - w.nch)] * vec[k];
      }
    }
  }
  // L x = y : root -> leaves; each dof publishes (x_d, x_parent, ...) for its children
  float x = 0.f;
  for (int lv = M.nlevel - 1; lv >= 0; --lv) {
    if (w.mylevel == lv) {
      float acc = y;
      float xa[MC];
#pragma unroll
      for (int c = 1; c < MC; ++c) {
        xa[c] = 0.f;
        if (c < w.nch) { xa[c] = xch[w.parent * MC + c - 1]; acc -= R[c] * xa[c]; }
      }
      x = acc * invd;
      xch[lane * MC] = x;
#pragma unroll
      for (int c = 1; c < MC; ++c)
        if (c < w.nch) xch[lane * MC + c] = xa[c];
    }
    syncwarp();
  }
  return x;
}

// ---------------------------------------------------------------------------------
// "Star" solve: root chain (NR dofs, e.g. the floating base) + up to 4 hanging serial chains
// (legs, arms; <= NL dofs each).  Block elimination of  [[A_l, C_l],[C_l^T, B]] x = g  with the
// warp split into 4 groups of 8 lanes: group l owns chain l, lane j of the group owns column j
// of [C_l | g_l] (NR coupling columns + the right-hand side; NR + 1 <= 8):
//   every lane : A_l = R^T R (3x3 / 5x5, redundantly per group)        registers, unrolled
//   lane (l,j) : w_j = R^-T c_j ;  row j of  W^T [W | z]  via 8-lane shuffles
//   all lanes  : sum over chains (2 xor-shuffle stages), S = B - sum_l W^T W, all-gather of S
//                inside the group, Cholesky + solve of the NR x NR root block (redundantly)
//   group l    : x_l = R^-1 (z - W x_B)  (3 xor-shuffle stages over the columns)
// Replaces the level-scheduled factor/solve (27 warp barriers) by 3 barriers and a few hundred
// unrolled register instructions with short dependency chains.  Rrow: compact row of H.
// ---------------------------------------------------------------------------------
template <int NL, int NR, int MCU>
DEV float star_solve(WarpCtx& w, const float* Rrow, float g) {
  static_assert(NR + 1 <= 8, "root block + rhs must fit the 8 lanes of a group");
  const DevModel& M = *w.M;
  const int lane = w.lane;
  float* Hb = SM(L);
  float* vec = SM(vec);
  syncwarp();
#pragma unroll
  for (int c = 0; c < MCU; ++c)
    if (c < w.nch) Hb[lane * MC + c] = Rrow[c];
  vec[lane] = g;
  syncwarp();
  const int grp = lane >> 3, j = lane & 7, gbase = lane & ~7;
  const bool ischain = grp < M.star_nchain;
  const int len = ischain ? M.star_len[grp] : 0;
  const int leaf = ischain ? M.star_leaf[grp] : 0;
  const int att = ischain ? M.star_att[grp] : NR;
  // ---- gather: chain block A (whole group) and this lane's column of [C | g] -------------------
  float A[NL][NL], wv[NL];
  int dofs[NL];
#pragma unroll
  for (int p = 0; p < NL; ++p) {
    const bool on = p < len;
    const int dof = on ? M.chain_tab[leaf][p] : 0;
    dofs[p] = dof;
    const float* row = Hb + dof * MC;
#pragma unroll
    for (int p2 = p; p2 < NL; ++p2) A[p][p2] = (on && p2 < len) ? row[p2 - p] : (p2 == p ? 1.f : 0.f);
    float cv = 0.f;
    if (on && j < NR && j >= att) cv = row[(len - p) + (j - att)];
    if (on && j == NR) cv = vec[dof];
    wv[p] = cv;
  }
  // ---- A = R^T R (upper R in place), w = R^-T c ------------------------------------------------------
  float rinv[NL];
#pragma unroll
  for (int p = 0; p < NL; ++p) {
    float d = A[p][p];
#pragma unroll
    for (int k = 0; k < p; ++k) d -= A[k][p] * A[k][p];
    const float inv = rsqrtf(fmaxf(d, DIAL_MINVAL));
    rinv[p] = inv;
#pragma unroll
    for (int p2 = p + 1; p2 < NL; ++p2) {
      float v = A[p][p2];
#pragma unroll
      for (int k = 0; k < p; ++k) v -= A[k][p] * A[k][p2];
      A[p][p2] = v * inv;
    }
    float v = wv[p];
#pragma unroll
    for (int k = 0; k < p; ++k) v -= A[k][p] * wv[k];
    wv[p] = v * inv;
  }
  // ---- row j of W^T [W | z], summed over the chains ---------------------------------------------------
  float t[NR + 1];
#pragma unroll
  for (int j2 = 0; j2 <= NR; ++j2) {
    float acc = 0.f;
#pragma unroll
    for (int p = 0; p < NL; ++p) acc += wv[p] * shfl(wv[p], gbase + j2);
    t[j2] = acc;
  }
#pragma unroll
  for (int j2 = 0; j2 <= NR; ++j2) {
    t[j2] += shfl_xor(t[j2], 8);
    t[j2] += shfl_xor(t[j2], 16);
  }
  // ---- root block: lane j holds row j of S and rhs_j, then all-gather inside the group ---------------
  float srow[NR], rhs = 0.f;
  {
    const int jj = j < NR ? j : 0;
    const int dofj = M.star_root[jj];
#pragma unroll
    for (int a2 = 0; a2 < NR; ++a2) {
      const float b = (a2 >= jj) ? Hb[dofj * MC + (a2 - jj)] : Hb[M.star_root[a2] * MC + (jj - a2)];
      srow[a2] = b - t[a2];
    }
    rhs = vec[dofj] - t[NR];
  }
  float S_[NR][NR], xB[NR];
#pragma unroll
  for (int a = 0; a < NR; ++a) {
#pragma unroll
    for (int a2 = a; a2 < NR; ++a2) S_[a][a2] = shfl(srow[a2], gbase + a);
    xB[a] = shfl(rhs, gbase + a);
  }
  // S = U^T U, solve (every lane redundantly)
  float sinv[NR];
#pragma unroll
  for (int a = 0; a < NR; ++a) {
    float d = S_[a][a];
#pragma unroll
    for (int k = 0; k < a; ++k) d -= S_[k][a] * S_[k][a];
    const float inv = rsqrtf(fmaxf(d, DIAL_MINVAL));
    sinv[a] = inv;
#pragma unroll
    for (int a2 = a + 1; a2 < NR; ++a2) {
      float v = S_[a][a2];
#pragma unroll
      for (int k = 0; k < a; ++k) v -= S_[k][a] * S_[k][a2];
      S_[a][a2] = v * inv;
    }
    float v = xB[a];
#pragma unroll
    for (int k = 0; k < a; ++k) v -= S_[k][a] * xB[k];
    xB[a] = v * inv;
  }
#pragma unroll
  for (int a = NR - 1; a >= 0; --a) {
    float v = xB[a];
#pragma unroll
    for (int a2 = a + 1; a2 < NR; ++a2) v -= S_[a][a2] * xB[a2];
    xB[a] = v * sinv[a];
  }
  // ---- chain back-substitution: x_l = R^-1 (z - W x_B) ----------------------------------------------
  float xb_j = 0.f;
#pragma unroll
  for (int a = 0; a < NR; ++a) xb_j = (j == a) ? xB[a] : xb_j;
  float xl[NL];
#pragma unroll
  for (int p = 0; p < NL; ++p) {
    float v = (j < NR) ? wv[p] * xb_j : 0.f;
    v += shfl_xor(v, 1); v += shfl_xor(v, 2); v += shfl_xor(v, 4);
    xl[p] = shfl(wv[p], gbase + NR) - v;
  }
#pragma unroll
  for (int p = NL - 1; p >= 0; --p) {
    float v = xl[p];
#pragma unroll
    for (int p2 = p + 1; p2 < NL; ++p2) v -= A[p][p2] * xl[p2];
    xl[p] = v * rinv[p];
  }
  // ---- scatter back to the dof lanes -------------------------------------------------------------------
  syncwarp();
  if (j == 0) {
#pragma unroll
    for (int p = 0; p < NL; ++p)
      if (p < len) vec[dofs[p]] = xl[p];
  }
  if (lane == 0) {
#pragma unroll
    for (int a = 0; a < NR; ++a) vec[M.star_root[a]] = xB[a];
  }
  syncwarp();
  return vec[lane];
}

// NL == 0: generic tree (level-scheduled compact Cholesky); otherwise the star solve
template <int NL, int NR, int MCU>
DEV float tree_solve(WarpCtx& w, float* R, float g) {
  if constexpr (NL == 0) {
    float invd = 0.f;
    factor_LTL(w, R, invd);
    return solve_LTL(w, R, invd, g);
  } else {
    return star_solve<NL, NR, MCU>(w, R, g);
  }
}

// y = M x; Mrow = this lane's compact row of M (also published in SM(Mb)).  Uses SM(vec).
template <int MCU>
DEV float mul_M(WarpCtx& w, const float* Mrow, float x) {
  const DevModel& M = *w.M;
  const int lane = w.lane;
  const float* Mb = SM(Mb);
  float* vec = SM(vec);
  syncwarp();
  vec[lane] = x;
  syncwarp();
  float y = 0.f;
#pragma unroll
  for (int c = 0; c < MCU; ++c)
    if (c < w.nch) y += Mrow[c] * vec[w.chain[c]];
  for (int k = lane + 1; k <= lane + w.ndesc; ++k) y += Mb[k * MC + (M.dof_nchain[k] - w.nch)] * vec[k];
  return y;
}

// contact-edge rows times a dof vector: lane e returns J_e . x.  J rows are stored compactly
// along the chain of the contact body's last dof.  Uses SM(vec).
DEV float mul_J(WarpCtx& w, float x) {
  const DevModel& M = *w.M;
  const int lane = w.lane;
  const float* Jc = SM(J);
  float* vec = SM(vec);
  syncwarp();
  vec[lane] = x;
  syncwarp();
  float y = 0.f;
  if (lane < M.nedge) {
    const int kc = M.con_lastdof[lane >> 2];
    const int nk = M.dof_nchain[kc];
    for (int p = 0; p < nk; ++p) y += Jc[lane * MC + p] * vec[M.chain_tab[kc][p]];
  }
  return y;
}

// J^T f for the contact-edge rows: lane e holds f_e, lane d returns sum_e J[e][d] f_e.
DEV float mul_JT(WarpCtx& w, float f) {
  const DevModel& M = *w.M;
  const int lane = w.lane;
  const float* Jc = SM(J);
  float* frow = SM(frow);
  syncwarp();
  frow[lane] = f;
  syncwarp();
  float y = 0.f;
  if (w.nch > 0) {
    for (int c = 0; c < M.m.ncon; ++c) {
      const int kc = M.con_lastdof[c];
      if ((M.dof_ancmask[kc] >> lane) & 1u) {
        const int off = M.dof_nchain[kc] - w.nch;
#pragma unroll
        for (int e = 0; e < 4; ++e) y += Jc[(4 * c + e) * MC + off] * frow[4 * c + e];
      }
    }
  }
  return y;
}

// stiffness / damping / impedance of a constraint row (mjx constraint._kbi)
DEV void kbi(float timestep, const float* solref, const float* solimp, float pos,
             float& k, float& b, float& imp) {
  float timeconst = fmaxf(solref[0], 2.f * timestep), dampratio = solref[1];
  float dmin = fminf(fmaxf(solimp[0], DIAL_MINIMP), DIAL_MAXIMP);
  float dmax = fminf(fmaxf(solimp[1], DIAL_MINIMP), DIAL_MAXIMP);
  float width = fmaxf(DIAL_MINVAL, solimp[2]);
  float mid = fminf(fmaxf(solimp[3], DIAL_MINIMP), DIAL_MAXIMP);
  float power = fmaxf(1.f, solimp[4]);
  k = 1.f / (dmax * dmax * timeconst * timeconst * dampratio * dampratio);
  b = 2.f / (dmax * timeconst);
  if (solref[0] <= 0.f) k = -solref[0] / (dmax * dmax);
  if (solref[1] <= 0.f) b = -solref[1] / dmax;
  float x = fabsf(pos) / width;
  float y;
  if (power == 2.f) {  // the MuJoCo default; avoids four powf calls
    y = x < mid ? x * x / mid : 1.f - (1.f - x) * (1.f - x) / (1.f - mid);
  } else {
    float a_ = (1.f / powf(mid, power - 1.f)) * powf(x, power);
    float b_ = 1.f - (1.f / powf(1.f - mid, power - 1.f)) * powf(fmaxf(1.f - x, 0.f), power);
    y = x < mid ? a_ : b_;
  }
  imp = dmin + y * (dmax - dmin);
  imp = fminf(fmaxf(imp, dmin), dmax);
  if (x > 1.f) imp = dmax;
}

// ---------------------------------------------------------------------------------
// Newton solver state kept in registers
//   lane d (< nv)   : dof-vector elements + the joint-limit row of dof d (if any)
//   lane e (< nedge): contact pyramid edge row e
// ---------------------------------------------------------------------------------
struct Solver {
  float qacc, Ma, grad, search, qfs, qas;  // qfs = qfrc_smooth, qas = qacc_smooth
  float l_sign, l_D, l_aref, l_Jaref;      // limit row (lane = dof)
  float e_D, e_aref, e_Jaref;              // contact edge row (lane = edge)
  float gauss, cost, prev_cost, gradnorm2; // warp-uniform scalars
  float qfc;                               // qfrc_constraint (dense path, for eulerdamp)
};

// efc_force, qfrc_constraint, costs and the gradient (solver.py _update_constraint + grad)
DEV void update_constraint(WarpCtx& w, Solver& S) {
  float fl = (S.l_Jaref < 0.f) ? -S.l_D * S.l_Jaref : 0.f;
  float fe = (S.e_Jaref < 0.f) ? -S.e_D * S.e_Jaref : 0.f;
  float qfc = mul_JT(w, fe) + S.l_sign * fl;
  S.grad = S.Ma - S.qfs - qfc;
  float g = (S.Ma - S.qfs) * (S.qacc - S.qas);
  float c = ((S.l_Jaref < 0.f) ? S.l_D * S.l_Jaref * S.l_Jaref : 0.f)
          + ((S.e_Jaref < 0.f) ? S.e_D * S.e_Jaref * S.e_Jaref : 0.f);
  float g2 = S.grad * S.grad;
  warp_sum3(g, c, g2);
  S.gauss = 0.5f * g;
  S.prev_cost = S.cost;
  S.cost = 0.5f * c + S.gauss;
  S.gradnorm2 = g2;
}

// compact row of H = M + J^T D_active J for this lane's dof
template <int MCU>
DEV void build_H(WarpCtx& w, const Solver& S, const float* Mrow, float* R) {
  const DevModel& M = *w.M;
  const int lane = w.lane;
  const float* Jc = SM(J);
  float* frow = SM(frow);
  syncwarp();
  frow[lane] = (S.e_Jaref < 0.f) ? S.e_D : 0.f;
  syncwarp();
#pragma unroll
  for (int c = 0; c < MCU; ++c) R[c] = Mrow[c];
  if (w.nch > 0) {
    R[0] += (S.l_Jaref < 0.f) ? S.l_D : 0.f;  // limit rows are +-e_d: diagonal only
    for (int c_ = 0; c_ < M.m.ncon; ++c_) {
      const int kc = M.con_lastdof[c_];
      if ((M.dof_ancmask[kc] >> lane) & 1u) {
        const int off = M.dof_nchain[kc] - w.nch;
        for (int e = 4 * c_; e < 4 * c_ + 4; ++e) {
          const float de = frow[e];
          if (de != 0.f) {
            const float* Je = Jc + e * MC + off;
            const float a = de * Je[0];
#pragma unroll
            for (int c = 0; c < MCU; ++c)
              if (c < w.nch) R[c] += a * Je[c];
          }
        }
      }
    }
  }
}


// ---------------------------------------------------------------------------------
// Star-layout solver kernels (star variants NL > 0).  Rows of M, H = M + J^T D J and J are kept
// as [NRP root columns | CS columns of the row's own chain] (NRP, CS: NR, NL rounded up to 4):
// every inner product below has compile-time offsets, vector (128-bit) shared-memory loads and no
// table look-ups — the compact-chain code above spends a third of its instructions on index
// arithmetic.  Per lane i (= dof i): Rr[NR] = H[i][root a], Rc[NL] = H[i][own chain, depth q].
//   Ms / Hs   [pos][RS]   full symmetric rows of M / H at the star position of the dof
//   Js        [edge][RS]  contact pyramid rows: root part + the part on the contact's chain
//   xs        [npos]      a dof vector in star order (zero in the padding slots)
// ---------------------------------------------------------------------------------
template <int NL, int NR>
struct StarDims {
  static constexpr int NRP = (NR + 3) & ~3, CS = (NL + 3) & ~3, RS = NRP + CS;
};

// N floats (N <= 8, rounded up to whole float4 loads; the source is padded) from a 16-byte aligned address
template <int N>
DEV void ldv(const float* p, float* out) {
  F4 a = ld4(p);
  out[0] = a.x; if (N > 1) out[1] = a.y; if (N > 2) out[2] = a.z; if (N > 3) out[3] = a.w;
  if (N > 4) {
    F4 b = ld4(p + 4);
    out[4] = b.x; if (N > 5) out[5] = b.y; if (N > 6) out[6] = b.z; if (N > 7) out[7] = b.w;
  }
}
// publish a row [Rr | Rc] at p (RS floats, padding written as zero)
template <int NL, int NR>
DEV void star_store_row(float* p, const float* Rr, const float* Rc) {
  using SD = StarDims<NL, NR>;
  float t[SD::RS];
#pragma unroll
  for (int i = 0; i < SD::RS; ++i) t[i] = 0.f;
#pragma unroll
  for (int a = 0; a < NR; ++a) t[a] = Rr[a];
#pragma unroll
  for (int q = 0; q < NL; ++q) t[SD::NRP + q] = Rc[q];
#pragma unroll
  for (int i = 0; i < SD::RS; i += 4) st4(p + i, t[i], t[i + 1], t[i + 2], t[i + 3]);
}

// y = M x and (edge lanes) J x with one publication of x.  Mr/Mc: this lane's row of M.
template <int NL, int NR, bool WITH_M, bool WITH_J, class SH = ShapeRT>
DEV void star_mul_MJ(WarpCtx& w, const float* Mr, const float* Mc, float x, float& Mx, float& Jx) {
  using SD = StarDims<NL, NR>;
  const DevModel& M = *w.M;
  float* xs = SM(xs);
  const float* Ms = SM(Ms);
  syncwarp();
  if (w.s_chain >= -1) xs[w.s_pos] = x;
  syncwarp();
  float xr[SD::NRP], xc[SD::CS];
  ldv<NR>(xs, xr);
  ldv<NL>(xs + w.s_cb, xc);
  float y = 0.f;
  if (WITH_M) {
  // (independent partial sums: the fp32 pipe has a 4-cycle dependent-issue latency and only
  // ~3.5 warps per scheduler to hide it)
  float y0 = 0.f, y1 = 0.f, y2 = 0.f, y3 = 0.f;
#pragma unroll
  for (int a = 0; a < NR; ++a) { if (a & 1) y1 += Mr[a] * xr[a]; else y0 += Mr[a] * xr[a]; }
  if (w.s_chain >= 0) {
#pragma unroll
    for (int q = 0; q < NL; ++q) { if (q & 1) y3 += Mc[q] * xc[q]; else y2 += Mc[q] * xc[q]; }
  } else if (w.s_chain == -1) {
    // root dof: the coupling column, sum over every chain slot of M[slot dof][root a] x[slot dof]
    const float* col = Ms + SD::NRP * SD::RS + w.s_col;
    const int nslot = SH::nchain(M) * SD::CS;
    for (int s0 = 0; s0 < nslot; s0 += 4) {
      F4 xv = ld4(xs + SD::NRP + s0);
      y0 += col[(s0 + 0) * SD::RS] * xv.x; y1 += col[(s0 + 1) * SD::RS] * xv.y;
      y2 += col[(s0 + 2) * SD::RS] * xv.z; y3 += col[(s0 + 3) * SD::RS] * xv.w;
    }
  }
  y = (y0 + y1) + (y2 + y3);
  }
  Mx = y;
  if (WITH_J) {
    float j = 0.f;
    if (w.lane < SH::nedge(M)) {
      const float* row = SM(Js) + w.lane * SD::RS;
      float jr[SD::NRP], jc[SD::CS], xe[SD::CS];
      ldv<NR>(row, jr);
      ldv<NL>(row + SD::NRP, jc);
      ldv<NL>(xs + w.e_cb, xe);
      float j0 = 0.f, j1 = 0.f, j2 = 0.f;
#pragma unroll
      for (int a = 0; a < NR; ++a) { if (a & 1) j1 += jr[a] * xr[a]; else j0 += jr[a] * xr[a]; }
#pragma unroll
      for (int q = 0; q < NL; ++q) j2 += jc[q] * xe[q];
      j = (j0 + j1) + j2;
    }
    Jx = j;
  }
}

// J^T f: edge lane e holds f_e; dof lane returns sum_e J[e][my column] f_e
template <int NL, int NR, class SH = ShapeRT>
DEV float star_mul_JT(WarpCtx& w, float f) {
  using SD = StarDims<NL, NR>;
  const DevModel& M = *w.M;
  const float* Js = SM(Js);
  float* frow = SM(frow);
  syncwarp();
  frow[w.lane] = f;
  syncwarp();
  float y0 = 0.f, y1 = 0.f, y2 = 0.f, y3 = 0.f;   // independent partial sums (dependent-issue latency)
  const float* col = Js + w.s_col;
  for (int c = 0; c < SH::ncon(M); ++c) {
    const F4 fv = ld4(frow + 4 * c);
    if ((w.s_conmask >> c) & 1u) {
      const float* jc = col + 4 * c * SD::RS;
      y0 += jc[0] * fv.x; y1 += jc[SD::RS] * fv.y; y2 += jc[2 * SD::RS] * fv.z; y3 += jc[3 * SD::RS] * fv.w;
    }
  }
  return (y0 + y1) + (y2 + y3);
}

// H row of this lane: M + active limit + sum over active edges d_e j_e^T j_e
template <int NL, int NR, class SH = ShapeRT>
DEV void star_build_H(WarpCtx& w, const Solver& S, const float* Mr, const float* Mc, float* Rr, float* Rc) {
  using SD = StarDims<NL, NR>;
  const DevModel& M = *w.M;
  const float* Js = SM(Js);
  float* frow = SM(frow);
  syncwarp();
  frow[w.lane] = (S.e_Jaref < 0.f) ? S.e_D : 0.f;
  syncwarp();
#pragma unroll
  for (int a = 0; a < NR; ++a) Rr[a] = Mr[a];
#pragma unroll
  for (int q = 0; q < NL; ++q) Rc[q] = Mc[q];
  const float ld = (S.l_Jaref < 0.f) ? S.l_D : 0.f;   // limit rows are +-e_d: diagonal only
  if (w.s_chain >= 0) {
#pragma unroll
    for (int q = 0; q < NL; ++q) Rc[q] += (q == w.s_depth) ? ld : 0.f;
  } else if (w.s_chain == -1) {
#pragma unroll
    for (int a = 0; a < NR; ++a) Rr[a] += (a == w.s_depth) ? ld : 0.f;
  }
  for (int e = 0; e < SH::nedge(M); ++e) {
    const float de = frow[e];
    if (de == 0.f) continue;                           // warp-uniform
    const float* row = Js + e * SD::RS;
    const float je = ((w.s_conmask >> (e >> 2)) & 1u) ? row[w.s_col] : 0.f;
    const float al = de * je;
    float jr[SD::NRP], jc[SD::CS];
    ldv<NR>(row, jr);
    ldv<NL>(row + SD::NRP, jc);
#pragma unroll
    for (int a = 0; a < NR; ++a) Rr[a] += al * jr[a];
#pragma unroll
    for (int q = 0; q < NL; ++q) Rc[q] += al * jc[q];   // other chains / root lanes: al == 0 or Rc unused
  }
}

// Solve H x = g for the star structure (block elimination, see star_solve above); rows in the
// star layout are published once and gathered with compile-time offsets.
template <int NL, int NR, class SH = ShapeRT>
DEV float star_solve2(WarpCtx& w, const float* Rr, const float* Rc, float g) {
  using SD = StarDims<NL, NR>;
  static_assert(NR + 1 <= 8, "root block + rhs must fit the 8 lanes of a group");
  const DevModel& M = *w.M;
  const int lane = w.lane;
  float* Hs = SM(Hs);
  float* xs = SM(xs);
  syncwarp();
  if (w.s_chain >= -1) {
    star_store_row<NL, NR>(Hs + w.s_pos * SD::RS, Rr, Rc);
    xs[w.s_pos] = g;
  }
  syncwarp();
  const int grp = lane >> 3, j = lane & 7, gbase = lane & ~7;
  const bool ischain = grp < SH::nchain(M);
  const int len = ischain ? M.star_len[grp] : 0;
  const int cb = SD::NRP + grp * SD::CS;
  // ---- gather: chain block A (whole group) and this lane's column of [C | g] -------------------
  float A[NL][NL], wv[NL];
#pragma unroll
  for (int p = 0; p < NL; ++p) {
    const bool on = p < len;
    const float* row = Hs + (cb + p) * SD::RS;
    float rc[SD::CS];
    ldv<NL>(row + SD::NRP, rc);
#pragma unroll
    for (int p2 = p; p2 < NL; ++p2) A[p][p2] = (on && p2 < len) ? rc[p2] : (p2 == p ? 1.f : 0.f);
    float cv = 0.f;
    if (on && j < NR) cv = row[j];
    if (on && j == NR) cv = xs[cb + p];
    wv[p] = cv;
  }
  // ---- A = R^T R (upper R in place), w = R^-T c ------------------------------------------------------
  float rinv[NL];
#pragma unroll
  for (int p = 0; p < NL; ++p) {
    float d = A[p][p];
#pragma unroll
    for (int k = 0; k < p; ++k) d -= A[k][p] * A[k][p];
    const float inv = rsqrtf(fmaxf(d, DIAL_MINVAL));
    rinv[p] = inv;
#pragma unroll
    for (int p2 = p + 1; p2 < NL; ++p2) {
      float v = A[p][p2];
#pragma unroll
      for (int k = 0; k < p; ++k) v -= A[k][p] * A[k][p2];
      A[p][p2] = v * inv;
    }
    float v = wv[p];
#pragma unroll
    for (int k = 0; k < p; ++k) v -= A[k][p] * wv[k];
    wv[p] = v * inv;
  }
  // ---- row j of W^T [W | z], summed over the chains ---------------------------------------------------
  float t[NR + 1];
#pragma unroll
  for (int j2 = 0; j2 <= NR; ++j2) {
    float acc = 0.f;
#pragma unroll
    for (int p = 0; p < NL; ++p) acc += wv[p] * shfl(wv[p], gbase + j2);
    t[j2] = acc;
  }
#pragma unroll
  for (int j2 = 0; j2 <= NR; ++j2) {
    t[j2] += shfl_xor(t[j2], 8);
    t[j2] += shfl_xor(t[j2], 16);
  }
  // ---- root block: lane j holds row j of S and rhs_j, then all-gather inside the group ---------------
  float srow[NR], rhs = 0.f;
  {
    const int jj = j < NR ? j : 0;
    float br[SD::NRP];
    ldv<NR>(Hs + jj * SD::RS, br);
#pragma unroll
    for (int a2 = 0; a2 < NR; ++a2) srow[a2] = br[a2] - t[a2];
    rhs = xs[jj] - t[NR];
  }
  float S_[NR][NR], xB[NR];
#pragma unroll
  for (int a = 0; a < NR; ++a) {
#pragma unroll
    for (int a2 = a; a2 < NR; ++a2) S_[a][a2] = shfl(srow[a2], gbase + a);
    xB[a] = shfl(rhs, gbase + a);
  }
  float sinv[NR];
#pragma unroll
  for (int a = 0; a < NR; ++a) {
    float d = S_[a][a];
#pragma unroll
    for (int k = 0; k < a; ++k) d -= S_[k][a] * S_[k][a];
    const float inv = rsqrtf(fmaxf(d, DIAL_MINVAL));
    sinv[a] = inv;
#pragma unroll
    for (int a2 = a + 1; a2 < NR; ++a2) {
      float v = S_[a][a2];
#pragma unroll
      for (int k = 0; k < a; ++k) v -= S_[k][a] * S_[k][a2];
      S_[a][a2] = v * inv;
    }
    float v = xB[a];
#pragma unroll
    for (int k = 0; k < a; ++k) v -= S_[k][a] * xB[k];
    xB[a] = v * inv;
  }
#pragma unroll
  for (int a = NR - 1; a >= 0; --a) {
    float v = xB[a];
#pragma unroll
    for (int a2 = a + 1; a2 < NR; ++a2) v -= S_[a][a2] * xB[a2];
    xB[a] = v * sinv[a];
  }
  // ---- chain back-substitution: x_l = R^-1 (z - W x_B) ----------------------------------------------
  float xb_j = 0.f;
#pragma unroll
  for (int a = 0; a < NR; ++a) xb_j = (j == a) ? xB[a] : xb_j;
  float xl[NL];
#pragma unroll
  for (int p = 0; p < NL; ++p) {
    float v = (j < NR) ? wv[p] * xb_j : 0.f;
    v += shfl_xor(v, 1); v += shfl_xor(v, 2); v += shfl_xor(v, 4);
    xl[p] = shfl(wv[p], gbase + NR) - v;
  }
#pragma unroll
  for (int p = NL - 1; p >= 0; --p) {
    float v = xl[p];
#pragma unroll
    for (int p2 = p + 1; p2 < NL; ++p2) v -= A[p][p2] * xl[p2];
    xl[p] = v * rinv[p];
  }
  // ---- scatter back to the dof lanes (star order) ------------------------------------------------------
  syncwarp();
  if (j == 0 && ischain) {
#pragma unroll
    for (int p = 0; p < NL; ++p)
      if (p < len) xs[cb + p] = xl[p];
  }
  if (lane == 0) {
#pragma unroll
    for (int a = 0; a < NR; ++a) xs[a] = xB[a];
  }
  syncwarp();
  return w.s_chain >= -1 ? xs[w.s_pos] : 0.f;
}

// efc_force, qfrc_constraint, costs and the gradient in the star layout
template <int NL, int NR, class SH = ShapeRT>
DEV void star_update_constraint(WarpCtx& w, Solver& S) {
  float fl = (S.l_Jaref < 0.f) ? -S.l_D * S.l_Jaref : 0.f;
  float fe = (S.e_Jaref < 0.f) ? -S.e_D * S.e_Jaref : 0.f;
  float qfc = star_mul_JT<NL, NR, SH>(w, fe) + S.l_sign * fl;
  S.grad = S.Ma - S.qfs - qfc;
  float g = (S.Ma - S.qfs) * (S.qacc - S.qas);
  float c = ((S.l_Jaref < 0.f) ? S.l_D * S.l_Jaref * S.l_Jaref : 0.f)
          + ((S.e_Jaref < 0.f) ? S.e_D * S.e_Jaref * S.e_Jaref : 0.f);
  float g2 = S.grad * S.grad;
  warp_sum3(g, c, g2);
  S.gauss = 0.5f * g;
  S.prev_cost = S.cost;
  S.cost = 0.5f * c + S.gauss;
  S.gradnorm2 = g2;
}

struct LSPoint { float alpha, cost, d0, d1; };

// Bracket update of the line search.  Default: MJX's rule (solver._linesearch) — lo / hi move to their Newton
// successor whenever they are on the wrong side (lo.d0 > 0) OR the successor's derivative is larger, whichever
// its sign.  On a step that crosses a cone-zone boundary this can throw away a valid bracket, the search then
// returns "no improvement" and the solver stops unconverged (DESIGN.md 2).  -DDIAL_ROBUST_LS (opt-in, custom /
// experimental builds: scripts/build_exp.py, dial_mpc_b200.custom) keeps the bracket: a successor is accepted
// only while it stays on the same side of the minimum.  A documented deviation from the reference, like the
// NaN guards; the stock library is built without it.
#ifdef DIAL_ROBUST_LS
#define DIAL_LS_SWAP_LO(lo, nx) (((lo).d0 < (nx).d0) && ((nx).d0 < 0.f))
#define DIAL_LS_SWAP_HI(hi, nx) (((hi).d0 > (nx).d0) && ((nx).d0 > 0.f))
#else
#define DIAL_LS_SWAP_LO(lo, nx) (((lo).d0 > 0.f) || ((lo).d0 < (nx).d0))
#define DIAL_LS_SWAP_HI(hi, nx) (((hi).d0 < 0.f) || ((hi).d0 > (nx).d0))
#endif

// All-reduce of 6 values per lane: reduce-scatter over the lane bits 16 / 8 (each lane keeps half
// of its values and sends the other half), plain butterflies for the rest, then an all-gather —
// 17 shuffles + 11 adds instead of 30 + 30.  Every lane ends with the same six sums.
DEV void warp_allsum6(int lane, float* v) {
  const bool b16 = (lane & 16) != 0, b8 = (lane & 8) != 0;
  // xor 16: lanes with bit 16 clear keep (v0, v1, v2), the others (v3, v4, v5)
  float u0 = b16 ? v[3] : v[0], u1 = b16 ? v[4] : v[1], u2 = b16 ? v[5] : v[2];
  const float s0 = b16 ? v[0] : v[3], s1 = b16 ? v[1] : v[4], s2 = b16 ? v[2] : v[5];
  u0 += shfl_xor(s0, 16); u1 += shfl_xor(s1, 16); u2 += shfl_xor(s2, 16);
  // xor 8: of (u0, u1) keep one; u2 goes on as a plain butterfly
  float t = b8 ? u1 : u0;
  const float st = b8 ? u0 : u1;
  t += shfl_xor(st, 8); u2 += shfl_xor(u2, 8);
  t += shfl_xor(t, 4); u2 += shfl_xor(u2, 4);
  t += shfl_xor(t, 2); u2 += shfl_xor(u2, 2);
  t += shfl_xor(t, 1); u2 += shfl_xor(u2, 1);
  // t: total of value (b16 ? 3 : 0) + (b8 ? 1 : 0); u2: total of value (b16 ? 5 : 2)
  v[0] = shfl(t, 0); v[1] = shfl(t, 8); v[3] = shfl(t, 16); v[4] = shfl(t, 24);
  v[2] = shfl(u2, 0); v[5] = shfl(u2, 16);
}

// Per-lane quadratic coefficients of the 1-D cost along the search direction (limit row of the
// dof lane, pyramid edge row of the edge lane); constant during one line search.
struct LSRow { float lq0, lq1, lq2, eq0, eq1, eq2; };

// Evaluate the 1-D piecewise-quadratic cost at NA (<= 3) alphas at once.  The bracketing loop of
// the line search needs only the derivatives d0 / d1: with COST = false the cost sums are left
// out (a third of the warp reductions); the costs of the points that survive are evaluated once
// at the end with the same expressions, so the result equals MJX's, which carries them along.
template <int NA, bool COST>
DEV void ls_points(int lane, const Solver& S, const LSRow& K, float l_jv, float e_jv, const float* qg, const float* al, LSPoint* out) {
  float s[3 * NA];
#pragma unroll
  for (int i = 0; i < 3 * NA; ++i) s[i] = 0.f;
#pragma unroll
  for (int i = 0; i < NA; ++i) {
    if (S.l_Jaref + al[i] * l_jv < 0.f) { if (COST) s[3 * i] += K.lq0; s[3 * i + 1] += K.lq1; s[3 * i + 2] += K.lq2; }
    if (S.e_Jaref + al[i] * e_jv < 0.f) { if (COST) s[3 * i] += K.eq0; s[3 * i + 1] += K.eq1; s[3 * i + 2] += K.eq2; }
  }
  if constexpr ((NA == 3 && !COST) || (NA == 2 && COST)) {
    // six sums: transposed reduction
    float v[6];
    if constexpr (NA == 3) { v[0] = s[1]; v[1] = s[2]; v[2] = s[4]; v[3] = s[5]; v[4] = s[7]; v[5] = s[8]; }
    else { v[0] = s[0]; v[1] = s[1]; v[2] = s[2]; v[3] = s[3]; v[4] = s[4]; v[5] = s[5]; }
    warp_allsum6(lane, v);
    if constexpr (NA == 3) { s[1] = v[0]; s[2] = v[1]; s[4] = v[2]; s[5] = v[3]; s[7] = v[4]; s[8] = v[5]; }
    else { s[0] = v[0]; s[1] = v[1]; s[2] = v[2]; s[3] = v[3]; s[4] = v[4]; s[5] = v[5]; }
  } else {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int i = 0; i < 3 * NA; ++i)
        if (COST || (i % 3) != 0) s[i] += shfl_xor(s[i], o);
    }
  }
#pragma unroll
  for (int i = 0; i < NA; ++i) {
    float t0 = qg[0] + s[3 * i], t1 = qg[1] + s[3 * i + 1], t2 = qg[2] + s[3 * i + 2];
    float a = al[i];
    out[i].alpha = a;
    out[i].cost = COST ? a * a * t2 + a * t1 + t0 : 0.f;
    out[i].d0 = 2.f * a * t2 + t1;
    out[i].d1 = 2.f * t2 + (t2 == 0.f ? DIAL_MINVAL : 0.f);
  }
}

// MJX solver._linesearch given M.search (mv) and J.search (e_jv) of this lane's rows
template <class SH = ShapeRT>
DEV void linesearch_core(WarpCtx& w, Solver& S, float mv, float e_jv) {
  const DevModel& M = *w.M;
  const int nv = SH::nv(M);
  const float scale = M.m.meaninertia * (float)(nv > 1 ? nv : 1);
  float l_jv = S.l_sign * S.search;
  float ss = S.search * S.search, sMa = S.search * (S.Ma - S.qfs), sMv = S.search * mv;
  warp_sum3(ss, sMa, sMv);
  float gtol = M.m.tolerance * M.m.ls_tolerance * sqrtf(ss) * scale;
  float qg[3] = {S.gauss, sMa, 0.5f * sMv};
  LSRow K;
  K.lq0 = 0.5f * S.l_Jaref * S.l_Jaref * S.l_D; K.lq1 = l_jv * S.l_Jaref * S.l_D; K.lq2 = 0.5f * l_jv * l_jv * S.l_D;
  K.eq0 = 0.5f * S.e_Jaref * S.e_Jaref * S.e_D; K.eq1 = e_jv * S.e_Jaref * S.e_D; K.eq2 = 0.5f * e_jv * e_jv * S.e_D;
  LSPoint p0, lo, hi;
  float a1[1] = {0.f};
  ls_points<1, true>(w.lane, S, K, l_jv, e_jv, qg, a1, &p0);
  a1[0] = p0.alpha - p0.d0 / p0.d1;
  ls_points<1, false>(w.lane, S, K, l_jv, e_jv, qg, a1, &lo);
  if (lo.d0 < p0.d0) { hi = p0; } else { hi = lo; lo = p0; }
  bool swap = true;
#pragma unroll 1
  for (int it = 0; it < SH::ls_iterations(M); ++it) {
    bool done = !swap;
    done |= (lo.d0 < 0.f) && (lo.d0 > -gtol);
    done |= (hi.d0 > 0.f) && (hi.d0 < gtol);
    if (done) break;
    LSPoint pt[3];
    float a3[3] = {lo.alpha - lo.d0 / lo.d1, hi.alpha - hi.d0 / hi.d1, 0.5f * (lo.alpha + hi.alpha)};
    ls_points<3, false>(w.lane, S, K, l_jv, e_jv, qg, a3, pt);
    const LSPoint lo_next = pt[0], hi_next = pt[1], mid = pt[2];
    bool swap_lo_next = DIAL_LS_SWAP_LO(lo, lo_next);
    if (swap_lo_next) lo = lo_next;
    bool swap_lo_mid = (mid.d0 < 0.f) && (lo.d0 < mid.d0);
    if (swap_lo_mid) lo = mid;
    bool swap_hi_next = DIAL_LS_SWAP_HI(hi, hi_next);
    if (swap_hi_next) hi = hi_next;
    bool swap_hi_mid = (mid.d0 > 0.f) && (hi.d0 > mid.d0);
    if (swap_hi_mid) hi = mid;
    swap = swap_lo_next || swap_lo_mid || swap_hi_next || swap_hi_mid;
  }
  // costs of the two surviving points (same expressions MJX evaluates when it visits them)
  {
    LSPoint fin[2];
    float a2[2] = {lo.alpha, hi.alpha};
    ls_points<2, true>(w.lane, S, K, l_jv, e_jv, qg, a2, fin);
    lo.cost = fin[0].cost; hi.cost = fin[1].cost;
  }
  bool improved = (lo.cost < p0.cost) || (hi.cost < p0.cost);
  float alpha = (lo.cost < hi.cost) ? lo.alpha : hi.alpha;
  if (!improved) alpha = 0.f;
  // fused, as the kernels with a run-time contact count compile them: with the count fixed (ShapeFixed)
  // the compiler splits them into a multiply and an add, which round twice
  S.qacc = __fmaf_rn(alpha, S.search, S.qacc);
  S.Ma = __fmaf_rn(alpha, mv, S.Ma);
  S.l_Jaref += alpha * l_jv;
  S.e_Jaref += alpha * e_jv;
}

template <int MCU>
DEV void linesearch(WarpCtx& w, Solver& S, const float* Mrow) {
  float mv = mul_M<MCU>(w, Mrow, S.search);
  float e_jv = mul_J(w, S.search);
  linesearch_core(w, S, mv, e_jv);
}

// ---------------------------------------------------------------------------------
// Dense / elliptic-cone solver path (NL < 0): models whose contacts couple two moving bodies
// or use elliptic friction cones (allegro_reorient: 19 contacts, condim 3/6, nv = 22).  H is no
// longer tree-sparse, so M, H and the contact Jacobian are dense in shared memory:
//   lane d (< nv)   : dof vectors + the limit row of dof d, row d of M / H / the Cholesky factor
//   lane c (< ncon) : the contact's rows (<= 6: normal, 2 tangents, torsion, 2 rolling)
// Cone cost (MuJoCo primal, restated in oracle/mjx_oracle.py): with N = mu x0, T = |fri o x_1..|
// top (N >= mu T): 0; bottom (mu N + T <= 0): plain quadratic; middle: 0.5 Dm (N - mu T)^2.
// ---------------------------------------------------------------------------------
struct ConeLane {
  float x[6], D[6], aref[6], fri[5];
  float mu, Dm;
  int dim, r0;
  bool inst;
};

DEV void dense_mul_J(WarpCtx& w, const ConeLane& C, float xd, float* out) {
  // contact lane c returns J_c x (its <= 6 rows).  The instantiated contacts are few and the dofs
  // many, so every dof lane multiplies its column and the rows are summed by xor-shuffles (all
  // lanes busy) instead of one contact lane walking the 22 columns alone.
  const DevModel& M = *w.M;
  const int nv = M.m.nv, lane = w.lane;
  const float* Jd = SM(Jd);
  const int* cact = reinterpret_cast<const int*>(SM(cact));
#pragma unroll
  for (int i = 0; i < 6; ++i) out[i] = 0.f;
  const float xv = lane < nv ? xd : 0.f;
  const int col = lane < nv ? lane : 0, js = M.jd_stride;
  for (int c = 0; c < M.m.ncon; ++c) {
    if (!cact[c]) continue;   // warp-uniform
    const int r0 = M.con_row0[c], dim = M.con_dim[c];
    const int idx = M.con_colidx[c][col];
    float p[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) p[i] = (i < dim && idx >= 0) ? Jd[(r0 + i) * js + idx] * xv : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int i = 0; i < 6; ++i)
        if (i < dim) p[i] += shfl_xor(p[i], o);
    }
    if (lane == c) {
#pragma unroll
      for (int i = 0; i < 6; ++i) out[i] = p[i];
    }
  }
  (void)C;
}

// rows of G (same shape as J) times ... J^T f: contact lanes publish f, dof lanes gather
DEV float dense_mul_JT(WarpCtx& w, const ConeLane& C, const float* f) {
  const DevModel& M = *w.M;
  const int nv = M.m.nv, lane = w.lane;
  const float* Jd = SM(Jd);
  float* fr = SM(frow2);
  const int* cact = reinterpret_cast<const int*>(SM(cact));
  syncwarp();
  if (lane < M.m.ncon) {
#pragma unroll
    for (int i = 0; i < 6; ++i)
      if (i < C.dim) fr[C.r0 + i] = f[i];
  }
  syncwarp();
  float y = 0.f;
  if (lane < nv) {
    for (int c = 0; c < M.m.ncon; ++c) {
      if (!cact[c]) continue;
      const int r0 = M.con_row0[c], dim = M.con_dim[c];
      const int idx = M.con_colidx[c][lane];
      if (idx < 0) continue;
      for (int i = 0; i < dim; ++i) y += Jd[(r0 + i) * M.jd_stride + idx] * fr[r0 + i];
    }
  }
  return y;
}

// zone: 0 top, 1 middle, 2 bottom.  cost and force of one contact at rows x.
DEV int cone_eval(const ConeLane& C, const float* x, float& cost, float* force, float& N, float& T) {
  cost = 0.f;
#pragma unroll
  for (int i = 0; i < 6; ++i) force[i] = 0.f;
  N = 0.f; T = 0.f;
  if (!C.inst) return 0;
  if (C.dim == 1) {   // frictionless: plain inequality row
    if (x[0] < 0.f) { cost = 0.5f * C.D[0] * x[0] * x[0]; force[0] = -C.D[0] * x[0]; return 2; }
    return 0;
  }
  N = C.mu * x[0];
  float tt = 0.f;
#pragma unroll
  for (int i = 1; i < 6; ++i)
    if (i < C.dim) { float u = x[i] * C.fri[i - 1]; tt += u * u; }
  T = sqrtf(tt);
  const bool bottom = (T <= 0.f && N < 0.f) || (T > 0.f && C.mu * N + T <= 0.f);
  const bool middle = (T > 0.f) && (N < C.mu * T) && (C.mu * N + T > 0.f);
  if (bottom) {
#pragma unroll
    for (int i = 0; i < 6; ++i)
      if (i < C.dim) { cost += 0.5f * C.D[i] * x[i] * x[i]; force[i] = -C.D[i] * x[i]; }
    return 2;
  }
  if (middle) {
    const float NmT = N - C.mu * T;
    const float f0 = -C.Dm * NmT * C.mu;
    cost = 0.5f * C.Dm * NmT * NmT;
    force[0] = f0;
#pragma unroll
    for (int i = 1; i < 6; ++i)
      if (i < C.dim) force[i] = -(f0 / T) * (x[i] * C.fri[i - 1]) * C.fri[i - 1];
    return 1;
  }
  return 0;
}

DEV void dense_update_constraint(WarpCtx& w, Solver& S, const ConeLane& C) {
  float cc, f[6], N, T;
  cone_eval(C, C.x, cc, f, N, T);
  float fl = (S.l_Jaref < 0.f) ? -S.l_D * S.l_Jaref : 0.f;
  float qfc = dense_mul_JT(w, C, f) + S.l_sign * fl;
  S.qfc = qfc;
  S.grad = S.Ma - S.qfs - qfc;
  float g = (S.Ma - S.qfs) * (S.qacc - S.qas);
  float c = ((S.l_Jaref < 0.f) ? S.l_D * S.l_Jaref * S.l_Jaref : 0.f) + 2.f * cc;
  float g2 = S.grad * S.grad;
  warp_sum3(g, c, g2);
  S.gauss = 0.5f * g;
  S.prev_cost = S.cost;
  S.cost = 0.5f * c + S.gauss;
  S.gradnorm2 = g2;
}

// dense Cholesky H = L L^T with row `lane` of H / L in registers (NVD = nv at compile time, fully
// unrolled): column k of the factor needs row k broadcast from lane k (shuffles), no shared memory
// and no barriers.  Hrow[j], j <= lane: lower triangle of H on entry, of L on return.
template <int NVD>
DEV float dense_factor_solve(WarpCtx& w, float* Hrow, float g) {
  const int lane = w.lane;
#pragma unroll
  for (int k = 0; k < NVD; ++k) {
    // row k is final once columns < k are done: lane k holds L[k][0..k-1] and the pivot
    float piv = Hrow[k];
#pragma unroll
    for (int p = 0; p < k; ++p) {
      const float lkp = shfl(Hrow[p], k);       // L[k][p]
      if (lane >= k) piv -= Hrow[p] * lkp;      // lanes > k: L[i][p] * L[k][p]; lane k: L[k][p]^2
    }
    // lane k: piv = H[k][k] - sum L[k][p]^2 ; lanes > k: piv = H[i][k] - sum L[i][p] L[k][p]
    const float dk = sqrtf(fmaxf(shfl(piv, k), DIAL_MINVAL));
    Hrow[k] = (lane == k) ? dk : piv / dk;
  }
  float y = g;
#pragma unroll
  for (int k = 0; k < NVD; ++k) {        // L y = g
    const float yk = shfl(y, k) / shfl(Hrow[k], k);
    if (lane == k) y = yk;
    if (lane > k) y -= Hrow[k] * yk;
  }
#pragma unroll
  for (int k = NVD - 1; k >= 0; --k) {   // L^T x = y :  x_k = (y_k - sum_{i>k} L[i][k] x_i) / L[k][k]
    float t = (lane > k && lane < NVD) ? Hrow[k] * y : 0.f;
    t = warp_sum(t);
    const float xk = (shfl(y, k) - t) / shfl(Hrow[k], k);
    if (lane == k) y = xk;
  }
  return y;
}

// H = Md + J^T G with G = D o J (bottom-zone contacts) or Hc J_c (middle-zone cone Hessian)
template <int NVD>
DEV void dense_build_H(WarpCtx& w, const Solver& S, const ConeLane& C, float* Hrow) {
  const DevModel& M = *w.M;
  const int nv = M.m.nv, lane = w.lane;
  const float* Jd = SM(Jd);
  float* Gs = SM(Gd);     // G rows of ONE contact (6 x nv scratch)
  const float* Md = SM(Md);
  int* cact = reinterpret_cast<int*>(SM(cact));
  float* hcs = SM(hcs);   // 6x6 cone Hessian of the contact being expanded
  syncwarp();
  // contact lanes: zone of their cone (cact: 1 top = no curvature, 2 bottom, 3 middle) and, for
  // the middle zone, the analytic Hessian of 0.5 Dm mu^2 (x0 - T)^2, y_i = fri_i x_i, s = x0 - T
  float Hc[6][6];
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = 0; j < 6; ++j) Hc[i][j] = 0.f;
  if (lane < M.m.ncon) {
    float cc, f[6], N, T;
    const int zone = cone_eval(C, C.x, cc, f, N, T);
    cact[lane] = C.inst ? (zone == 2 ? 2 : zone == 1 ? 3 : 1) : 0;
    if (C.inst && zone == 1) {
      const float sc = C.Dm * C.mu * C.mu, s = C.x[0] - T, iT = 1.f / T;
      float y[6];
#pragma unroll
      for (int i = 1; i < 6; ++i) y[i] = (i < C.dim) ? C.x[i] * C.fri[i - 1] : 0.f;
      Hc[0][0] = sc;
#pragma unroll
      for (int i = 1; i < 6; ++i) {
        if (i < C.dim) {
          Hc[0][i] = Hc[i][0] = -sc * C.fri[i - 1] * y[i] * iT;
#pragma unroll
          for (int j = 1; j < 6; ++j)
            if (j < C.dim)
              Hc[i][j] = sc * C.fri[i - 1] * C.fri[j - 1] * (y[i] * y[j] * iT * iT * (1.f + s * iT) - (i == j ? s * iT : 0.f));
        }
      }
    }
  }
  syncwarp();
  // H rows: lane i holds H[i][0..i].  Start from M + the active limit row, then add J_c^T G_c for
  // every curved contact: G_c (<= 6 x nv) is formed in a small scratch with one dof column per lane
  // (the contacts are few, the dofs many) and consumed at once, so no nrow x nv copy of G exists.
#pragma unroll
  for (int j = 0; j < NVD; ++j) Hrow[j] = 0.f;
  if (lane < nv) {
#pragma unroll
    for (int j = 0; j < NVD; ++j) Hrow[j] = (j <= lane) ? Md[lane * nv + j] : 0.f;
#pragma unroll
    for (int j = 0; j < NVD; ++j)
      if (j == lane) Hrow[j] += (S.l_Jaref < 0.f) ? S.l_D : 0.f;
  }
  for (int c = 0; c < M.m.ncon; ++c) {
    const int z = cact[c];   // warp-uniform
    if (z < 2) continue;
    const int r0 = M.con_row0[c], dim = M.con_dim[c];
    if (z == 3 && lane == c) {
#pragma unroll
      for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) hcs[i * 6 + j] = Hc[i][j];
    }
    syncwarp();   // hcs published; previous contact's Gs fully consumed
    float Dc[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) Dc[i] = shfl(C.D[i], c);
    float jc[6];
    const int idx = lane < nv ? M.con_colidx[c][lane] : -1;
#pragma unroll
    for (int i = 0; i < 6; ++i) jc[i] = (i < dim && idx >= 0) ? Jd[(r0 + i) * M.jd_stride + idx] : 0.f;
    if (lane < nv) {
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        if (i < dim) {
          float a;
          if (z == 2) {
            a = Dc[i] * jc[i];
          } else {
            a = 0.f;
#pragma unroll
            for (int j = 0; j < 6; ++j) a += hcs[i * 6 + j] * jc[j];
          }
          Gs[i * nv + lane] = a;
        }
      }
    }
    syncwarp();
    if (lane < nv) {
      for (int i = 0; i < dim; ++i) {
        const float a = jc[i];
        const float* Gr = Gs + i * nv;
#pragma unroll
        for (int j = 0; j < NVD; ++j) Hrow[j] += a * Gr[j];
      }
    }
  }
  syncwarp();
}

// dense M x (lane = dof)
DEV float dense_mul_M(WarpCtx& w, float x) {
  const int nv = w.M->m.nv, lane = w.lane;
  const float* Md = SM(Md);
  float* vec = SM(vec);
  syncwarp();
  vec[lane] = x;
  syncwarp();
  float y = 0.f;
  if (lane < nv)
    for (int j = 0; j < nv; ++j) y += Md[(j <= lane ? lane * nv + j : j * nv + lane)] * vec[j];
  return y;
}

// Per-lane coefficients of the 1-D cost along the search direction; constant during one line
// search (mjx solver._linesearch evaluates them inside every point; hoisted here).
struct LSCoef {
  float q0, q1, q2;                       // limit row of this dof lane: quadratic in alpha
  float Q0, Q1, Q2, UU, UV, VV, U0, V0;   // cone of this contact lane (mjx _eval_pt_elliptic)
};

DEV LSCoef dense_ls_coef(const Solver& S, const ConeLane& C, float l_jv, const float* cv) {
  LSCoef K;
  K.q0 = 0.5f * S.l_Jaref * S.l_Jaref * S.l_D; K.q1 = l_jv * S.l_Jaref * S.l_D; K.q2 = 0.5f * l_jv * l_jv * S.l_D;
  K.Q0 = K.Q1 = K.Q2 = K.UU = K.UV = K.VV = 0.f;
  if (C.inst) {
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      if (i < C.dim) {
        K.Q0 += 0.5f * C.x[i] * C.x[i] * C.D[i]; K.Q1 += cv[i] * C.x[i] * C.D[i]; K.Q2 += 0.5f * cv[i] * cv[i] * C.D[i];
        if (i > 0) {
          const float f2 = C.fri[i - 1] * C.fri[i - 1];
          K.UU += C.x[i] * C.x[i] * f2; K.UV += C.x[i] * cv[i] * f2; K.VV += cv[i] * cv[i] * f2;
        }
      }
    }
  }
  K.U0 = C.mu * C.x[0]; K.V0 = C.mu * cv[0];
  return K;
}

// line-search points: derivatives (and, with COST, the cost) at NA alphas (limit rows + cones).
// The bracketing loop needs only d0 / d1; the costs of the surviving points are evaluated once
// at the end (same expressions), which removes a third of the warp reductions.
template <int NA, bool COST>
DEV void dense_ls_points(int lane, const Solver& S, const ConeLane& C, const LSCoef& K, float l_jv, const float* cv,
                         const float* qg, const float* al, LSPoint* out) {
  float s[3 * NA];
#pragma unroll
  for (int i = 0; i < 3 * NA; ++i) s[i] = 0.f;
#pragma unroll
  for (int i = 0; i < NA; ++i)
    if (S.l_Jaref + al[i] * l_jv < 0.f) {
      if (COST) s[3 * i] += al[i] * al[i] * K.q2 + al[i] * K.q1 + K.q0;
      s[3 * i + 1] += 2.f * al[i] * K.q2 + K.q1;
      s[3 * i + 2] += 2.f * K.q2;
    }
  if (C.inst) {
#pragma unroll
    for (int i = 0; i < NA; ++i) {
      const float a = al[i];
      if (C.dim == 1) {
        if (C.x[0] + a * cv[0] < 0.f) {
          if (COST) s[3 * i] += a * a * K.Q2 + a * K.Q1 + K.Q0;
          s[3 * i + 1] += 2.f * a * K.Q2 + K.Q1; s[3 * i + 2] += 2.f * K.Q2;
        }
        continue;
      }
      const float N = K.U0 + a * K.V0;
      const float Tsq = K.UU + a * (2.f * K.UV + a * K.VV);
      const float T = sqrtf(fmaxf(Tsq, 0.f));
      const bool bottom = (Tsq <= 0.f && N < 0.f) || (Tsq > 0.f && C.mu * N + T <= 0.f);
      const bool middle = (Tsq > 0.f) && (N < C.mu * T) && (C.mu * N + T > 0.f);
      if (bottom) {
        if (COST) s[3 * i] += a * a * K.Q2 + a * K.Q1 + K.Q0;
        s[3 * i + 1] += 2.f * a * K.Q2 + K.Q1; s[3 * i + 2] += 2.f * K.Q2;
      } else if (middle) {
        const float iT = 1.f / T;
        const float T1 = (K.UV + a * K.VV) * iT;
        const float T2 = (K.VV - T1 * T1) * iT;   // VV/T - (UV + a VV) T1 / T^2
        const float NmT = N - C.mu * T, dN = K.V0 - C.mu * T1;
        if (COST) s[3 * i] += 0.5f * C.Dm * NmT * NmT;
        s[3 * i + 1] += C.Dm * NmT * dN;
        s[3 * i + 2] += C.Dm * (dN * dN + NmT * (-C.mu * T2));
      }
    }
  }
  if constexpr ((NA == 3 && !COST) || (NA == 2 && COST)) {
    float v[6];   // six sums: transposed reduction (17 shuffles instead of 30)
    if constexpr (NA == 3) { v[0] = s[1]; v[1] = s[2]; v[2] = s[4]; v[3] = s[5]; v[4] = s[7]; v[5] = s[8]; }
    else { v[0] = s[0]; v[1] = s[1]; v[2] = s[2]; v[3] = s[3]; v[4] = s[4]; v[5] = s[5]; }
    warp_allsum6(lane, v);
    if constexpr (NA == 3) { s[1] = v[0]; s[2] = v[1]; s[4] = v[2]; s[5] = v[3]; s[7] = v[4]; s[8] = v[5]; }
    else { s[0] = v[0]; s[1] = v[1]; s[2] = v[2]; s[3] = v[3]; s[4] = v[4]; s[5] = v[5]; }
  } else {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int i = 0; i < 3 * NA; ++i)
        if (COST || (i % 3) != 0) s[i] += shfl_xor(s[i], o);
    }
  }
#pragma unroll
  for (int i = 0; i < NA; ++i) {
    const float a = al[i];
    out[i].alpha = a;
    out[i].cost = COST ? a * a * qg[2] + a * qg[1] + qg[0] + s[3 * i] : 0.f;
    out[i].d0 = 2.f * a * qg[2] + qg[1] + s[3 * i + 1];
    const float d1 = 2.f * qg[2] + s[3 * i + 2];
    out[i].d1 = d1 + (d1 == 0.f ? DIAL_MINVAL : 0.f);
  }
}

DEV void dense_linesearch(WarpCtx& w, Solver& S, ConeLane& C) {
  const DevModel& M = *w.M;
  const int nv = M.m.nv;
  const float scale = M.m.meaninertia * (float)(nv > 1 ? nv : 1);
  float mv = dense_mul_M(w, S.search);
  float cv[6];
  dense_mul_J(w, C, S.search, cv);
  float l_jv = S.l_sign * S.search;
  float ss = S.search * S.search, sMa = S.search * (S.Ma - S.qfs), sMv = S.search * mv;
  warp_sum3(ss, sMa, sMv);
  float gtol = M.m.tolerance * M.m.ls_tolerance * sqrtf(ss) * scale;
  float qg[3] = {S.gauss, sMa, 0.5f * sMv};
  const LSCoef K = dense_ls_coef(S, C, l_jv, cv);
  LSPoint p0, lo, hi;
  float a1[1] = {0.f};
  dense_ls_points<1, true>(w.lane, S, C, K, l_jv, cv, qg, a1, &p0);
  a1[0] = p0.alpha - p0.d0 / p0.d1;
  dense_ls_points<1, false>(w.lane, S, C, K, l_jv, cv, qg, a1, &lo);
  if (lo.d0 < p0.d0) { hi = p0; } else { hi = lo; lo = p0; }
  bool swap = true;
  // In fp32 the bracket can rarely reach `gtol` (the derivative noise is orders of magnitude above
  // it), so MJX's loop burns its whole budget on a sequence that has become periodic: an iteration
  // is a deterministic function of (lo, hi, swap).  Brent's cycle detection finds the period;
  // the state after the full `ls_iterations` is then reached by running only the remainder
  // modulo the period — bit-identical result, typically 10-20 iterations instead of 50.
  LSPoint snap_lo = lo, snap_hi = hi;
  bool snap_swap = swap;
  int snap_it = 0, power = 1, stop_at = M.m.ls_iterations;
  int it = 0;
  for (; it < stop_at; ++it) {
    bool done = !swap;
    done |= (lo.d0 < 0.f) && (lo.d0 > -gtol);
    done |= (hi.d0 > 0.f) && (hi.d0 < gtol);
    if (done) break;
#ifndef DIAL_NO_LS_CYCLE   // (tests build the emulator both ways and compare bit for bit)
    if (stop_at == M.m.ls_iterations && it > 0) {
      const bool same = swap == snap_swap && lo.alpha == snap_lo.alpha && hi.alpha == snap_hi.alpha &&
                        lo.d0 == snap_lo.d0 && hi.d0 == snap_hi.d0 && lo.d1 == snap_lo.d1 && hi.d1 == snap_hi.d1;
      if (same) {
        const int period = it - snap_it;
        stop_at = it + (M.m.ls_iterations - it) % period;
        if (it >= stop_at) break;
      } else if (it - snap_it == power) {
        snap_lo = lo; snap_hi = hi; snap_swap = swap; snap_it = it; power *= 2;
      }
    }
#endif
    LSPoint pt[3];
    float a3[3] = {lo.alpha - lo.d0 / lo.d1, hi.alpha - hi.d0 / hi.d1, 0.5f * (lo.alpha + hi.alpha)};
    dense_ls_points<3, false>(w.lane, S, C, K, l_jv, cv, qg, a3, pt);
    const LSPoint lo_next = pt[0], hi_next = pt[1], mid = pt[2];
    bool swap_lo_next = DIAL_LS_SWAP_LO(lo, lo_next);
    if (swap_lo_next) lo = lo_next;
    bool swap_lo_mid = (mid.d0 < 0.f) && (lo.d0 < mid.d0);
    if (swap_lo_mid) lo = mid;
    bool swap_hi_next = DIAL_LS_SWAP_HI(hi, hi_next);
    if (swap_hi_next) hi = hi_next;
    bool swap_hi_mid = (mid.d0 > 0.f) && (hi.d0 > mid.d0);
    if (swap_hi_mid) hi = mid;
    swap = swap_lo_next || swap_lo_mid || swap_hi_next || swap_hi_mid;
  }
  DIAL_TRACE(w.lane, 1, it);
  // costs of the two surviving points (mjx carries them along; same expressions, evaluated once)
  {
    LSPoint fin[2];
    float a2[2] = {lo.alpha, hi.alpha};
    dense_ls_points<2, true>(w.lane, S, C, K, l_jv, cv, qg, a2, fin);
    lo.cost = fin[0].cost; hi.cost = fin[1].cost;
  }
  bool improved = (lo.cost < p0.cost) || (hi.cost < p0.cost);
  float alpha = (lo.cost < hi.cost) ? lo.alpha : hi.alpha;
  if (!improved) alpha = 0.f;
  S.qacc += alpha * S.search;
  S.Ma += alpha * mv;
  S.l_Jaref += alpha * l_jv;
#pragma unroll
  for (int i = 0; i < 6; ++i) C.x[i] += alpha * cv[i];
}

// sections 8-9 of the physics step for the dense path; returns qacc (and qacc_int: the one the
// integrator uses, = qacc without eulerdamp), leaves S.qfc
template <int NVD>
DEV float dense_constraint_solve(WarpCtx& w, Solver& S, const float* Mrow, float myqvel, float& qacc_int) {
  const DevModel& M = *w.M;
  const dial_model_desc& m = M.m;
  const int lane = w.lane, nv = m.nv, d = lane;
  const bool isdof = d < nv;
  float* Jd = SM(Jd);
  float* Md = SM(Md);
  const float* cdof = SM(cdof);
  const float* rcom = SM(rcom);
  const float* cdist = SM(cdist);
  const float* cpos = SM(cpos);
  const float* cframe = SM(cframe);
  const float* qpos = SM(qpos);
  int* cact = reinterpret_cast<int*>(SM(cact));
  // dense M (lower triangle) from the compact rows
  if (isdof) {
    for (int j = 0; j <= d; ++j) Md[d * nv + j] = 0.f;
#pragma unroll
    for (int c = 0; c < MC; ++c)
      if (c < w.nch) Md[d * nv + w.chain[c]] = Mrow[c];
  }
  // contact rows: Jacobian columns (lane = dof), frame @ (jac(b2) - jac(b1))
  if (lane < m.ncon) {
    const int k = M.con_pair[lane];
    cact[lane] = (cdist[lane] - (m.pair_margin[k] - m.pair_gap[k]) < 0.f) ? 1 : 0;
  }
  syncwarp();
  if (isdof) {
    V3 ca_ = ld3(cdof + CDS * d), cl_ = ld3(cdof + CDS * d + 3);
    V3 rc = ld3(rcom + 3 * M.body_rootidx[m.dof_bodyid[d]]);
    for (int c = 0; c < m.ncon; ++c) {
      if (!cact[c]) continue;
      const int k = M.con_pair[c];
      const int b1 = m.geom_bodyid[m.pair_geom1[k]], b2 = m.geom_bodyid[m.pair_geom2[k]];
      const float sgn = (float)((M.body_dofmask[b2] >> d) & 1u) - (float)((M.body_dofmask[b1] >> d) & 1u);
      const int r0 = M.con_row0[c], dim = M.con_dim[c];
      const int idx = M.con_colidx[c][d];
      if (idx < 0) continue;   // sgn == 0: dof d moves both bodies or neither
      V3 jp = (cl_ + cross(ca_, ld3(cpos + 3 * c) - rc)) * sgn, jr = ca_ * sgn;
      for (int i = 0; i < dim; ++i) {
        V3 fr = ld3(cframe + 9 * c + 3 * (i % 3));
        Jd[(r0 + i) * M.jd_stride + idx] = dot(fr, i < 3 ? jp : jr);
      }
    }
    // joint-limit row of this dof
    int lj = M.dof_limited[d];
    if (lj >= 0) {
      float qv = qpos[m.jnt_qposadr[lj]];
      float dmin = qv - m.jnt_range[lj][0], dmax = m.jnt_range[lj][1] - qv;
      float pos = fminf(dmin, dmax) - m.jnt_margin[lj];
      if (pos < 0.f) {
        float sign = dmin < dmax ? 1.f : -1.f;
        float k_, b_, imp;
        kbi(m.timestep, m.jnt_solref[lj], m.jnt_solimp[lj], pos, k_, b_, imp);
        float Rr = fmaxf(m.dof_invweight0[d] * (1.f - imp) / imp, DIAL_MINVAL);
        S.l_sign = sign;
        S.l_D = 1.f / Rr;
        S.l_aref = -b_ * (sign * myqvel) - k_ * imp * pos;
      }
    }
  }
  // per-contact row data (lane = contact)
  ConeLane C;
#pragma unroll
  for (int i = 0; i < 6; ++i) { C.x[i] = 0.f; C.D[i] = 0.f; C.aref[i] = 0.f; }
#pragma unroll
  for (int i = 0; i < 5; ++i) C.fri[i] = 0.f;
  C.mu = 0.f; C.Dm = 0.f; C.dim = 0; C.r0 = 0; C.inst = false;
  if (lane < m.ncon) {
    C.dim = M.con_dim[lane]; C.r0 = M.con_row0[lane];
    C.inst = cact[lane] != 0;
  }
  float jq[6];
  dense_mul_J(w, C, myqvel, jq);
  if (C.inst) {
    const int k = M.con_pair[lane];
    const int b1 = m.geom_bodyid[m.pair_geom1[k]], b2 = m.geom_bodyid[m.pair_geom2[k]];
    const float pos = cdist[lane] - (m.pair_margin[k] - m.pair_gap[k]);
    const float t = m.body_invweight0[b1] + m.body_invweight0[b2];
#pragma unroll
    for (int i = 0; i < 5; ++i) C.fri[i] = m.pair_friction[k][i];
    float k_, b_, imp;
    kbi(m.timestep, m.pair_solref[k], m.pair_solimp[k], pos, k_, b_, imp);
    const float Rn = fmaxf(t * (1.f - imp) / imp, DIAL_MINVAL);
    C.D[0] = 1.f / Rn;
    C.aref[0] = -b_ * jq[0] - k_ * imp * pos;
#pragma unroll
    for (int i = 1; i < 6; ++i) {
      if (i < C.dim) {
        const float Ri = fmaxf(Rn / m.impratio * C.fri[0] * C.fri[0] / (C.fri[i - 1] * C.fri[i - 1]), DIAL_MINVAL);
        C.D[i] = 1.f / Ri;
        C.aref[i] = -b_ * jq[i];
      }
    }
    C.mu = C.fri[0] * rsqrtf(m.impratio);
    C.Dm = C.D[0] / fmaxf(C.mu * C.mu * (1.f + C.mu * C.mu), DIAL_MINVAL);
  }

  // ---- qacc_smooth, warm-start choice, Newton iterations (solver.solve) ------------------------
  const float scale = m.meaninertia * (float)(nv > 1 ? nv : 1);
  const float mywarm = isdof ? SM(warm)[d] : 0.f;
  syncwarp();
  // ONE factor/solve site for the three linear systems of the step (the unrolled register
  // Cholesky is ~8.6 k SASS instructions per inlined copy: three copies were 45 % of the kernel):
  //   mode 0: M x = qfrc_smooth            -> qacc_smooth, warm-start choice
  //   mode 1: H(active set) x = grad       -> Newton direction, line search          (solver.solve)
  //   mode 2: (M + dt diag(damping)) x = qfrc_smooth + qfrc_constraint               (eulerdamp)
  float Hrow[NVD];
#pragma unroll
  for (int j = 0; j < NVD; ++j) Hrow[j] = (isdof && j <= d) ? Md[d * nv + j] : (j == d ? 1.f : 0.f);
  float g = S.qfs;
  int mode = 0, it = 0;
  bool done = false;
  qacc_int = 0.f;
  for (;;) {
    float x = 0.f;
    if (mode != 1 || !done) x = dense_factor_solve<NVD>(w, Hrow, g);
    if (mode == 2) { qacc_int = x; break; }
    if (mode == 0) {
      S.qas = x;
      float xw[6], xs[6], cw, cs, f[6], N, T;
      float Maw = dense_mul_M(w, mywarm);
      dense_mul_J(w, C, mywarm, xw);
      dense_mul_J(w, C, S.qas, xs);
#pragma unroll
      for (int i = 0; i < 6; ++i) { xw[i] -= C.aref[i]; xs[i] -= C.aref[i]; }
      cone_eval(C, xw, cw, f, N, T);
      cone_eval(C, xs, cs, f, N, T);
      float lJw = S.l_sign * mywarm - S.l_aref, lJs = S.l_sign * S.qas - S.l_aref;
      float gw = (Maw - S.qfs) * (mywarm - S.qas);
      float tw = ((lJw < 0.f) ? S.l_D * lJw * lJw : 0.f) + 2.f * cw;
      float ts = ((lJs < 0.f) ? S.l_D * lJs * lJs : 0.f) + 2.f * cs;
      warp_sum3(gw, tw, ts);
      const bool usewarm = (0.5f * tw + 0.5f * gw) < (0.5f * ts);
      S.qacc = usewarm ? mywarm : S.qas;
      S.Ma = usewarm ? Maw : S.qfs;
      S.l_Jaref = usewarm ? lJw : lJs;
#pragma unroll
      for (int i = 0; i < 6; ++i) C.x[i] = usewarm ? xw[i] : xs[i];
      S.cost = INFINITY;
      S.prev_cost = 0.f;
      mode = 1;
    } else if (!done) {
      S.search = -x;
      dense_linesearch(w, S, C);
      ++it;
    }
    if (!done) {
      dense_update_constraint(w, S, C);
      done = it >= m.iterations;
      if (m.iterations != 1 || it > 0) {
        float improvement = (S.prev_cost - S.cost) / scale;
        float gradient = sqrtf(S.gradnorm2) / scale;
        if (m.iterations != 1) done = done || (improvement < m.tolerance) || (gradient < m.tolerance);
      }
      // a diverged sample (NaN / inf cost) can never satisfy the convergence tests: stop instead of
      // burning iterations x ls_iterations on it (its result is garbage either way, weight 0 later)
      if (!(fabsf(S.cost) <= 3.0e38f)) done = true;
    }
    // lock-step level 3: the warps of the CTA start every Newton iteration together (shared
    // instruction fetch inside the solver); a finished warp keeps arriving until all are done
    const bool any = w.itersync ? cta_sync_or(!done) : !done;
    if (!any) {
      if (!m.eulerdamp) { qacc_int = S.qacc; break; }
      mode = 2;   // implicit joint damping: (M + dt diag(damping))^-1 (qfrc_smooth + qfrc_constraint)
#pragma unroll
      for (int j = 0; j < NVD; ++j) Hrow[j] = (isdof && j <= d) ? Md[d * nv + j] : 0.f;
#pragma unroll
      for (int j = 0; j < NVD; ++j)
        if (j == d) Hrow[j] += isdof ? m.timestep * m.dof_damping[d] : 1.f;
      g = S.qfs + S.qfc;
      continue;
    }
    if (done) continue;
    dense_build_H<NVD>(w, S, C, Hrow);
    g = S.grad;
  }
#ifndef DIAL_HOST_EMUL
  if (w.dbg && lane == 0) { atomicAdd(w.dbg, 1.f); atomicAdd(w.dbg + 1, (float)it); }
#endif
  DIAL_TRACE(lane, 0, it);
  return S.qacc;
}

// ---------------------------------------------------------------------------------
// collision (lane = contact): MJX collision_primitive plane-sphere, plane-capsule (2 contacts),
// sphere-sphere, sphere-capsule, capsule-capsule; fixed-size contact arrays.
// ---------------------------------------------------------------------------------
DEV V3 mat_z(const float* X, const float* q) {   // z axis of  X * quat_to_mat(q)
  float Rg[9];
  qmat(ldq(q), Rg);
  return v3(X[0] * Rg[2] + X[1] * Rg[5] + X[2] * Rg[8], X[3] * Rg[2] + X[4] * Rg[5] + X[5] * Rg[8],
            X[6] * Rg[2] + X[7] * Rg[5] + X[8] * Rg[8]);
}
DEV V3 mat_apply(const float* X, const float* p) {
  return v3(X[0] * p[0] + X[1] * p[1] + X[2] * p[2], X[3] * p[0] + X[4] * p[1] + X[5] * p[2],
            X[6] * p[0] + X[7] * p[1] + X[8] * p[2]);
}
DEV V3 vnormalize(V3 a, float& n) {
  n = sqrtf(dot(a, a));
  return a * (1.f / (n + 1e-6f * (n == 0.f ? 1.f : 0.f)));
}
DEV V3 closest_segment_point(V3 a, V3 b, V3 pt) {
  V3 ab = b - a;
  float t = dot(pt - a, ab) / (dot(ab, ab) + 1e-6f);
  return a + ab * fminf(fmaxf(t, 0.f), 1.f);
}
DEV void closest_segment_to_segment(V3 a0, V3 a1, V3 b0, V3 b1, V3& pa, V3& pb) {
  float len_a, len_b;
  V3 dir_a = vnormalize(a1 - a0, len_a), dir_b = vnormalize(b1 - b0, len_b);
  float ha = 0.5f * len_a, hb = 0.5f * len_b;
  V3 a_mid = a0 + dir_a * ha, b_mid = b0 + dir_b * hb;
  V3 trans = a_mid - b_mid;
  float dd = dot(dir_a, dir_b), dat = dot(dir_a, trans), dbt = dot(dir_b, trans);
  float denom = 1.f - dd * dd;
  float ta = (-dat + dd * dbt) / (denom + 1e-6f);
  float tb = dbt + ta * dd;
  ta = fminf(fmaxf(ta, -ha), ha);
  tb = fminf(fmaxf(tb, -hb), hb);
  V3 best_a = a_mid + dir_a * ta, best_b = b_mid + dir_b * tb;
  V3 new_a = closest_segment_point(a0, a1, best_b), new_b = closest_segment_point(b0, b1, best_a);
  V3 e1 = new_a - best_b, e2 = new_b - best_a;
  if (dot(e1, e1) < dot(e2, e2)) { pa = new_a; pb = best_b; } else { pa = best_a; pb = new_b; }
}
DEV V3 frame_tangent(V3 n) {   // second row of mjx math.make_frame(n)
  V3 alt = (n.y > -0.5f && n.y < 0.5f) ? v3(0, 1, 0) : v3(0, 0, 1);
  float bn;
  return vnormalize(alt - n * dot(n, alt), bn);
}

// A floor contact on a terrain: the plane of the triangle under the sphere centre c replaces the floor's, as
// its normal n and the point org = (c.x, c.y, H) on it.  A flat triangle gives exactly the floor's normal
// (0, 0, 1), so a flat terrain at the floor's height computes bitwise what the floor computes.
DEV void terrain_plane(const DevTerrain& T, V3 c, V3& n, V3& org) {
  float sx, sy;
  const float H = terrain_at(T, c.x, c.y, sx, sy);
  n = (sx == 0.f && sy == 0.f) ? v3(0.f, 0.f, 1.f) : v3(-sx, -sy, 1.f) * (1.f / sqrtf(1.f + sx * sx + sy * sy));
  org = v3(c.x, c.y, H);
}

template <class SH = ShapeRT>
DEV void collide(WarpCtx& w) {
  const DevModel& M = *w.M;
  const dial_model_desc& m = M.m;
  const int lane = w.lane;
  if (lane >= SH::ncon(M)) return;
  const float* xpos = SM(xpos);
  const float* xmat = SM(xmat);
  const int k = M.con_pair[lane];
  const int g1 = m.pair_geom1[k], g2 = m.pair_geom2[k];
  const int b1 = m.geom_bodyid[g1], b2 = m.geom_bodyid[g2];
  const float* X1 = xmat + 9 * b1;
  const float* X2 = xmat + 9 * b2;
  const V3 gp1 = mat_apply(X1, m.geom_pos[g1]) + ld3(xpos + 3 * b1);
  const V3 gp2 = mat_apply(X2, m.geom_pos[g2]) + ld3(xpos + 3 * b2);
  const int kind = SH::pair_kind(M, k);
  V3 n, t1, p;
  float dist;
  if (kind == PAIR_PLANE_SPHERE || kind == PAIR_PLANE_CAPSULE) {
    n = mat_z(X1, m.geom_quat[g1]);
    const float radius = m.geom_size[g2][0];
    V3 center = gp2, org = gp1;
    if (kind == PAIR_PLANE_CAPSULE) {
      V3 ax = mat_z(X2, m.geom_quat[g2]);
#ifdef DIAL_TERRAIN
      // this end sphere's own triangle, before the frame is built from n (the same centre is computed again
      // below, where the flat builds compute it: moving that line changes their register allocation)
      center = gp2 + ax * ((M.con_sub[lane] == 0 ? 1.f : -1.f) * m.geom_size[g2][1]);
      if (w.ter && b1 == 0) terrain_plane(*w.ter, center, n, org);
#endif
      float bn;
      V3 bd = vnormalize(ax - n * dot(n, ax), bn);
      V3 alt = (n.y > -0.5f && n.y < 0.5f) ? v3(0, 1, 0) : v3(0, 0, 1);
      t1 = bn < 0.5f ? alt : bd;
      center = gp2 + ax * ((M.con_sub[lane] == 0 ? 1.f : -1.f) * m.geom_size[g2][1]);
    } else {
#ifdef DIAL_TERRAIN
      if (w.ter && b1 == 0) terrain_plane(*w.ter, center, n, org);
#endif
      t1 = frame_tangent(n);
    }
    dist = dot(center - org, n) - radius;
    p = center - n * (radius + 0.5f * dist);
  } else {
    V3 q1 = gp1, q2 = gp2;
    if (kind == PAIR_SPHERE_CAPSULE) {
      V3 seg = mat_z(X2, m.geom_quat[g2]) * m.geom_size[g2][1];
      q2 = closest_segment_point(gp2 - seg, gp2 + seg, gp1);
    } else if (kind == PAIR_CAPSULE_CAPSULE) {
      V3 s1 = mat_z(X1, m.geom_quat[g1]) * m.geom_size[g1][1];
      V3 s2 = mat_z(X2, m.geom_quat[g2]) * m.geom_size[g2][1];
      closest_segment_to_segment(gp1 - s1, gp1 + s1, gp2 - s2, gp2 + s2, q1, q2);
    }
    float dn;
    n = vnormalize(q2 - q1, dn);
    if (dn == 0.f) n = v3(1, 0, 0);
    const float r1 = m.geom_size[g1][0], r2 = m.geom_size[g2][0];
    dist = dn - (r1 + r2);
    p = q1 + n * (r1 + 0.5f * dist);
    float nn;
    n = vnormalize(n, nn);
    t1 = frame_tangent(n);
  }
  SM(cdist)[lane] = dist;
  st3(SM(cpos) + 3 * lane, p);
  st3(SM(cframe) + 9 * lane, n);
  st3(SM(cframe) + 9 * lane + 3, t1);
  st3(SM(cframe) + 9 * lane + 6, cross(n, t1));
}

// ---------------------------------------------------------------------------------
// one physics step (mjx.step) for the warp's sample.  State (qpos,qvel,warm,ctrl) in
// the slab; kinematic arrays of the forward pass are left in the slab for the reward.
// ---------------------------------------------------------------------------------
template <int NL, int NR, class SH = ShapeRT>
DEV void physics_step(WarpCtx& w, bool integrate) {
  constexpr int MCU = (NL == 3 && NR == 6) ? 9 : DIAL_MAXCHAIN;  // longest dof chain of the variant
  const DevModel& M = *w.M;
  const dial_model_desc& m = M.m;
  const int lane = w.lane, nb = SH::nbody(M), nv = SH::nv(M);
  float* xpos = SM(xpos); float* xquat = SM(xquat); float* xmat = SM(xmat); float* xipos = SM(xipos);
  float* cinert = SM(cinert); float* cdof = SM(cdof); float* cdofdot = SM(cdofdot);
  float* cvel = SM(cvel); float* cacc = SM(cacc); float* cfrc = SM(cfrc);
  float* J = SM(J);
  float* qpos = SM(qpos); float* qvel = SM(qvel); float* warm = SM(warm); float* ctrl = SM(ctrl);
  float* cpos = SM(cpos); float* cframe = SM(cframe); float* cdist = SM(cdist); float* rcom = SM(rcom);

  // ---- 1. kinematics (lane = body) -----------------------------------------------------------
  // Everything that does not depend on the parent is done for all bodies at once, before and after
  // the level loop: the transform of the body w.r.t. its parent frame (joint rotation included)
  //   quat = normalize(pq * qL), pos = ppos + rot(pq, pL), anchor = ppos + rot(pq, aL), axis = rot(pq, axL)
  // and, afterwards, the rotation matrices and the inertial frame.  The loop only composes.
  const int b = lane;
  const bool isbody = b > 0 && b < nb;
  const int depth = isbody ? m.body_depth[b] : -1;
  const int jid = isbody ? m.body_jntadr[b] : -1;
  const int jtype = jid >= 0 ? m.jnt_type[jid] : -1;
  V3 anchor = v3(0, 0, 0), axis = v3(0, 0, 1), xip = v3(0, 0, 0);
  float ximat[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) ximat[i] = 0.f;
  Q4 qL; qL.w = 1.f; qL.x = qL.y = qL.z = 0.f;
  V3 pL = v3(0, 0, 0), aL = v3(0, 0, 0), axL = v3(0, 0, 1);
  if (isbody) {
    const Q4 bq = ldq(m.body_quat[b]);
    const V3 bp = ld3(m.body_pos[b]);
    qL = bq; pL = bp;
    if (jtype == JNT_HINGE || jtype == JNT_SLIDE) {
      const int qa = m.jnt_qposadr[jid];
      const V3 jp = ld3(m.jnt_pos[jid]), ja = ld3(m.jnt_axis[jid]);
      aL = bp + qrot(bq, jp);
      axL = qrot(bq, ja);
      const float dq = qpos[qa] - m.qpos0[qa];
      if (jtype == JNT_HINGE) {
        qL = qmul(bq, axisangle(ja, dq));
        pL = aL - qrot(qL, jp);
      } else {
        pL = bp + axL * dq;
      }
    }
  }
  V3 pos = v3(0, 0, 0);
  Q4 quat; quat.w = 1.f; quat.x = quat.y = quat.z = 0.f;
  for (int lv = 1; lv <= SH::maxdepth(M); ++lv) {
    if (depth == lv) {
      if (jtype == JNT_FREE) {
        const int qa = m.jnt_qposadr[jid];
        pos = ld3(qpos + qa);
        quat = qnormalize(ldq(qpos + qa + 3));
        stq(qpos + qa + 3, quat);
        anchor = pos;
        axis = v3(0, 0, 1);
      } else {
        const int p = m.body_parentid[b];
        const Q4 pq = ldq(xquat + 4 * p);
        const V3 pp = ld3(xpos + 3 * p);
        quat = qmul(pq, qL);
        pos = pp + qrot(pq, pL);
        anchor = pp + qrot(pq, aL);
        axis = qrot(pq, axL);
      }
      quat = qnormalize(quat);
      st3(xpos + 3 * b, pos);
      stq(xquat + 4 * b, quat);
    }
    syncwarp();
  }
  if (isbody) {
    float R[9];
    qmat(quat, R);
#pragma unroll
    for (int i = 0; i < 9; ++i) xmat[9 * b + i] = R[i];
    xip = pos + qrot(quat, ld3(m.body_ipos[b]));
    st3(xipos + 3 * b, xip);
    qmat(qmul(quat, ldq(m.body_iquat[b])), ximat);
  }

  // ---- 2. subtree COM of each tree root --------------------------------------------
  const int myroot = isbody ? M.body_rootidx[b] : -1;
  V3 com = v3(0, 0, 0);
  for (int r = 0; r < SH::nroot(M); ++r) {
    float mass = (myroot == r) ? m.body_mass[b] : 0.f;
    float sx = mass * xip.x, sy = mass * xip.y, sz = mass * xip.z;
    warp_sum3(sx, sy, sz);
    V3 c = v3(sx, sy, sz) * M.root_invmass[r];
    if (lane == 0) st3(rcom + 3 * r, c);
    if (myroot == r) com = c;
  }

  // ---- 3. cinert (lane = body) and cdof (lane = jointed body) -------------------------
  if (isbody) {
    V3 off = xip - com;
    float mass = m.body_mass[b];
    const float* di = m.body_inertia[b];
    float I[6];  // xx yy zz xy xz yz of  R diag R^T
    I[0] = ximat[0] * ximat[0] * di[0] + ximat[1] * ximat[1] * di[1] + ximat[2] * ximat[2] * di[2];
    I[1] = ximat[3] * ximat[3] * di[0] + ximat[4] * ximat[4] * di[1] + ximat[5] * ximat[5] * di[2];
    I[2] = ximat[6] * ximat[6] * di[0] + ximat[7] * ximat[7] * di[1] + ximat[8] * ximat[8] * di[2];
    I[3] = ximat[0] * ximat[3] * di[0] + ximat[1] * ximat[4] * di[1] + ximat[2] * ximat[5] * di[2];
    I[4] = ximat[0] * ximat[6] * di[0] + ximat[1] * ximat[7] * di[1] + ximat[2] * ximat[8] * di[2];
    I[5] = ximat[3] * ximat[6] * di[0] + ximat[4] * ximat[7] * di[1] + ximat[5] * ximat[8] * di[2];
    float o2 = dot(off, off);
    float* ci = cinert + CIS * b;
    st4(ci, I[0] + mass * (o2 - off.x * off.x), I[1] + mass * (o2 - off.y * off.y), I[2] + mass * (o2 - off.z * off.z),
        I[3] - mass * off.x * off.y);
    st4(ci + 4, I[4] - mass * off.x * off.z, I[5] - mass * off.y * off.z, mass * off.x, mass * off.y);
    st2(ci + 8, mass * off.z, mass);
    if (jid >= 0) {
      int d = m.jnt_dofadr[jid];
      V3 offset = com - anchor;
      if (jtype == JNT_FREE) {
        for (int i = 0; i < 3; ++i) {
          float* c0 = cdof + CDS * (d + i);
          st4(c0, 0.f, 0.f, 0.f, i == 0 ? 1.f : 0.f);
          st2(c0 + 4, i == 1 ? 1.f : 0.f, i == 2 ? 1.f : 0.f);
          V3 ax = v3(xmat[9 * b + i], xmat[9 * b + 3 + i], xmat[9 * b + 6 + i]);
          V3 cx = cross(ax, offset);
          float* c1 = cdof + CDS * (d + 3 + i);
          st4(c1, ax.x, ax.y, ax.z, cx.x);
          st2(c1 + 4, cx.y, cx.z);
        }
      } else if (jtype == JNT_HINGE) {
        V3 cx = cross(axis, offset);
        st4(cdof + CDS * d, axis.x, axis.y, axis.z, cx.x);
        st2(cdof + CDS * d + 4, cx.y, cx.z);
      } else {
        st4(cdof + CDS * d, 0.f, 0.f, 0.f, axis.x);
        st2(cdof + CDS * d + 4, axis.y, axis.z);
      }
    }
  }
  syncwarp();

  // ---- 4. velocities / accelerations down the tree, local RNE force ---------------------
  float mycv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, myca[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int lv = 1; lv <= SH::maxdepth(M); ++lv) {
    if (depth == lv) {
      int p = m.body_parentid[b];
      float cv[6], ca[6];
#pragma unroll
      for (int i = 0; i < 6; ++i) { cv[i] = cvel[6 * p + i]; ca[i] = cacc[6 * p + i]; }
      if (jtype == JNT_FREE) {
        int d = m.jnt_dofadr[jid];
        for (int k = 0; k < 3; ++k) {
          float qd = qvel[d + k], cd[6];
          ld6(cdof + CDS * (d + k), cd);
#pragma unroll
          for (int i = 0; i < 6; ++i) cv[i] += cd[i] * qd;
          st4(cdofdot + CDS * (d + k), 0.f, 0.f, 0.f, 0.f);
          st2(cdofdot + CDS * (d + k) + 4, 0.f, 0.f);
        }
        float cvt[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) cvt[i] = cv[i];
        for (int k = 3; k < 6; ++k) {
          float dd[6], cd[6];
          ld6(cdof + CDS * (d + k), cd);
          mcross(cvt, cd, dd);
          float qd = qvel[d + k];
          st6(cdofdot + CDS * (d + k), dd);
#pragma unroll
          for (int i = 0; i < 6; ++i) {
            cv[i] += cd[i] * qd;
            ca[i] += dd[i] * qd;
          }
        }
      } else if (jid >= 0) {
        int d = m.jnt_dofadr[jid];
        float dd[6], cd[6];
        ld6(cdof + CDS * d, cd);
        mcross(cv, cd, dd);
        float qd = qvel[d];
        st6(cdofdot + CDS * d, dd);
#pragma unroll
        for (int i = 0; i < 6; ++i) {
          cv[i] += cd[i] * qd;
          ca[i] += dd[i] * qd;
        }
      }
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        cvel[6 * b + i] = cv[i];
        cacc[6 * b + i] = ca[i];
        mycv[i] = cv[i]; myca[i] = ca[i];
      }
    }
    syncwarp();
  }
  // local RNE force of every body at once (needs only the body's own velocity / acceleration)
  if (isbody) {
    float f1[6], f2[6], f3[6], cib[10];
    ld10(cinert + CIS * b, cib);
    inert_mul(cib, myca, f1);
    inert_mul(cib, mycv, f2);
    mcross_force(mycv, f2, f3);
#pragma unroll
    for (int i = 0; i < 6; ++i) cfrc[6 * b + i] = f1[i] + f3[i];
  }
  syncwarp();

  // ---- 5. composite inertia and RNE force of every subtree ---------------------------------
  // Bodies are in depth-first order, so the subtree of b is the index range [b, b + ndesc_b].
  // 16 component lanes (10 of crb, 6 of cfrc) x 2 bodies per pass; no level loop, no barriers.
  {
    float* crb = SM(crb);
    float* cfs = SM(cfs);
    const int comp = lane & 15, half = lane >> 4;
    const float* src = comp < 10 ? cinert + comp : cfrc + (comp - 10);
    const int stride = comp < 10 ? CIS : 6;
    float* dst = comp < 10 ? crb + comp : cfs + (comp - 10);
    if (NL > 0 && SH::sb_on(M)) {
      // star models: suffix sums along each hanging chain (half-warp h takes chains h and h + 2),
      // then the root bodies, deepest first, collect their child root and the chains hanging off them
      for (int l = half; l < SH::nchain(M); l += 2) {
        const int top = M.sb_top[l];
        float acc = 0.f;
        for (int k = SH::sb_len(M, l) - 1; k >= 0; --k) { acc += src[(top + k) * stride]; dst[(top + k) * stride] = acc; }
      }
      syncwarp();
      if (half == 0) {
        float below = 0.f;
        for (int r = 0; r < SH::sb_nroot(M); ++r) {
          float acc = src[M.sb_root[r] * stride] + below;
          for (int l = 0; l < SH::nchain(M); ++l)
            if (M.sb_att[l] == r) acc += dst[M.sb_top[l] * stride];
          dst[M.sb_root[r] * stride] = acc;
          below = acc;
        }
      }
    } else {
      for (int b0 = 1; b0 < nb; b0 += 2) {
        const int bb = b0 + half;
        if (bb < nb) {
          float acc = 0.f;
          const int last = bb + M.body_ndesc[bb];
          for (int jb = bb; jb <= last; ++jb) acc += src[jb * stride];
          dst[bb * stride] = acc;
        }
      }
    }
  }
  syncwarp();

  // ---- 7. collision (lane = contact) ---------------------------------------------------
  collide<SH>(w);
  syncwarp();

  // ---- 6. compact mass-matrix row, bias, smooth force (lane = dof) ----------------------
  Solver S;
  S.qfs = 0.f; S.qas = 0.f;
  S.l_sign = 0.f; S.l_D = 0.f; S.l_aref = 0.f; S.l_Jaref = 0.f;
  S.e_D = 0.f; S.e_aref = 0.f; S.e_Jaref = 0.f;
  S.qacc = S.Ma = S.grad = S.search = 0.f;
  S.gauss = S.cost = S.prev_cost = S.gradnorm2 = 0.f;
  S.qfc = 0.f;
  const int d = lane;
  const bool isdof = d < nv;
  float myqvel = isdof ? qvel[d] : 0.f;
  float mycdof[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // this lane's cdof row, kept for the contact Jacobian
  constexpr bool STAR = NL > 0;   // star layout rows (Mr | Mc) instead of compact chain rows
  constexpr int SNR = STAR ? NR : 1, SNL = STAR ? NL : 1;
  float Mrow[STAR ? 1 : MC], R[STAR ? 1 : MC];
  float Mr[SNR], Mc[SNL], Rr[SNR], Rc[SNL];
#pragma unroll
  for (int a = 0; a < SNR; ++a) { Mr[a] = 0.f; Rr[a] = 0.f; }
#pragma unroll
  for (int q = 0; q < SNL; ++q) { Mc[q] = 0.f; Rc[q] = 0.f; }
  if constexpr (!STAR) {
#pragma unroll
    for (int c = 0; c < MCU; ++c) { Mrow[c] = 0.f; R[c] = 0.f; }
  }
  if (isdof) {
    int bi = m.dof_bodyid[d];
    float f[6];
    {
      float crbb[10];
      ld10(SM(crb) + CIS * bi, crbb);
      ld6(cdof + CDS * d, mycdof);
      inert_mul(crbb, mycdof, f);
    }
    if constexpr (STAR) {
      using SD = StarDims<NL, NR>;
      // row of M in the star layout: entries towards ancestors are computed (CRB), the others
      // are the mirror images of other lanes' entries (filled below from the published rows)
      const float arm = m.dof_armature[d];
      if (w.s_chain >= 0) {
        const int att = M.star_att[w.s_chain];
#pragma unroll
        for (int q = 0; q < NL; ++q)
          if (q <= w.s_depth) { float cd[6]; ld6(cdof + CDS * (w.s_top + q), cd); Mc[q] = dot6(f, cd) + (q == w.s_depth ? arm : 0.f); }
#pragma unroll
        for (int a = 0; a < NR; ++a)
          if (a >= att) { float cd[6]; ld6(cdof + CDS * M.star_root[a], cd); Mr[a] = dot6(f, cd); }
      } else {
#pragma unroll
        for (int a = 0; a < NR; ++a)
          if (a >= w.s_depth) { float cd[6]; ld6(cdof + CDS * M.star_root[a], cd); Mr[a] = dot6(f, cd) + (a == w.s_depth ? arm : 0.f); }
      }
      star_store_row<NL, NR>(SM(Ms) + w.s_pos * SD::RS, Mr, Mc);
    } else {
#pragma unroll
      for (int c = 0; c < MCU; ++c)
        if (c < w.nch) { float cd[6]; ld6(cdof + CDS * w.chain[c], cd); Mrow[c] = dot6(f, cd); }
      Mrow[0] += m.dof_armature[d];
      if constexpr (NL >= 0) {   // the dense path keeps M in SM(Md) instead
        float* Mb = SM(Mb);
#pragma unroll
        for (int c = 0; c < MCU; ++c)
          if (c < w.nch) Mb[d * MC + c] = Mrow[c];
      }
    }
    float bias = dot6(mycdof, SM(cfs) + 6 * bi);
    float act = 0.f;
    int a = M.dof_actuator[d];
    if (a >= 0) {
      float c = ctrl[a];
      if (m.actuator_ctrllimited[a]) c = fminf(fmaxf(c, m.actuator_ctrlrange[a][0]), m.actuator_ctrlrange[a][1]);
      float force = m.actuator_gain[a] * c + m.actuator_bias[a][0]
                  + m.actuator_bias[a][1] * qpos[m.actuator_qposadr[a]] + m.actuator_bias[a][2] * myqvel;
      if (m.actuator_forcelimited[a]) force = fminf(fmaxf(force, m.actuator_forcerange[a][0]), m.actuator_forcerange[a][1]);
      act = force * m.actuator_gear[a];
    }
    S.qfs = -m.dof_damping[d] * myqvel - bias + act;
  }
  if constexpr (NL >= 0) {
    if (M.s_on && M.o_crb == M.o_Hs) {   // crb / cfs overlay the star H rows (dial_host.h): hand them back zeroed
      syncwarp();
      float* z = SM(crb);
      for (int i = lane; i < (CIS + 6) * nb; i += 32) z[i] = 0.f;
      syncwarp();
    }
  }
  if constexpr (STAR) {
    using SD = StarDims<NL, NR>;
    float* Ms = SM(Ms);
    syncwarp();
    if (w.s_chain >= 0) {          // entries towards deeper dofs of my chain
#pragma unroll
      for (int q = 0; q < NL; ++q)
        if (q > w.s_depth) { Mc[q] = Ms[(w.s_cb + q) * SD::RS + SD::NRP + w.s_depth]; Ms[w.s_pos * SD::RS + SD::NRP + q] = Mc[q]; }
    } else if (w.s_chain == -1) {  // entries towards deeper root dofs
#pragma unroll
      for (int a = 0; a < NR; ++a)
        if (a < w.s_depth) { Mr[a] = Ms[a * SD::RS + w.s_depth]; Ms[w.s_pos * SD::RS + a] = Mr[a]; }
    }
  }

  float qacc, qacc_int;
  if constexpr (NL < 0) {
    if (w.midsync) cta_sync();   // lock-step CTAs: enter the constraint solve together
    else syncwarp();             // crb / cfs may overlay SM(Md), which the solve writes (dial_host.h)
    qacc = dense_constraint_solve<NR>(w, S, Mrow, myqvel, qacc_int);   // also the eulerdamp solve (mode 2)
  } else if constexpr (STAR) {
  using SD = StarDims<NL, NR>;
  // ---- 8. constraint rows in the star layout (lane = dof writes its column of every row) --------
  float* Js = SM(Js);
  if (isdof) {
    V3 ca_ = v3(mycdof[0], mycdof[1], mycdof[2]), cl_ = v3(mycdof[3], mycdof[4], mycdof[5]);
    V3 rc = ld3(rcom + 3 * M.body_rootidx[m.dof_bodyid[d]]);
    for (int c = 0; c < SH::ncon(M); ++c) {
      if (!((w.s_conmask >> c) & 1u)) continue;   // my column is structurally zero in this contact's rows
      const int k = M.con_pair[c];
      float e0 = 0.f, e1 = 0.f, e2 = 0.f, e3 = 0.f;
      const bool moves = (M.body_dofmask[m.geom_bodyid[m.pair_geom2[k]]] >> d) & 1u;
      if (moves && cdist[c] - (m.pair_margin[k] - m.pair_gap[k]) < 0.f) {
        V3 p = ld3(cpos + 3 * c);
        V3 jp = cl_ + cross(ca_, p - rc);
        float jn = dot(ld3(cframe + 9 * c), jp), j1 = dot(ld3(cframe + 9 * c + 3), jp), j2 = dot(ld3(cframe + 9 * c + 6), jp);
        float mu0 = m.pair_friction[k][0], mu1 = m.pair_friction[k][1];
        e0 = jn + mu0 * j1; e1 = jn - mu0 * j1; e2 = jn + mu1 * j2; e3 = jn - mu1 * j2;
      }
      float* col = Js + 4 * c * SD::RS + w.s_col;
      col[0] = e0; col[SD::RS] = e1; col[2 * SD::RS] = e2; col[3 * SD::RS] = e3;
    }
    int lj = M.dof_limited[d];
    if (lj >= 0) {
      float qv = qpos[m.jnt_qposadr[lj]];
      float dmin = qv - m.jnt_range[lj][0], dmax = m.jnt_range[lj][1] - qv;
      float pos = fminf(dmin, dmax) - m.jnt_margin[lj];
      if (pos < 0.f) {
        float sign = dmin < dmax ? 1.f : -1.f;
        float k_, b_, imp;
        kbi(m.timestep, m.jnt_solref[lj], m.jnt_solimp[lj], pos, k_, b_, imp);
        float Rr_ = fmaxf(m.dof_invweight0[d] * (1.f - imp) / imp, DIAL_MINVAL);
        S.l_sign = sign;
        S.l_D = 1.f / Rr_;
        S.l_aref = -b_ * (sign * myqvel) - k_ * imp * pos;
      }
    }
  }
  float ejv, dummy;
  star_mul_MJ<NL, NR, false, true, SH>(w, Mr, Mc, myqvel, dummy, ejv);
  if (lane < SH::nedge(M)) {
    int c = lane >> 2;
    int k = M.con_pair[c];
    float pos = cdist[c] - (m.pair_margin[k] - m.pair_gap[k]);
    if (pos < 0.f) {
      int b1 = m.geom_bodyid[m.pair_geom1[k]], b2 = m.geom_bodyid[m.pair_geom2[k]];
      float mu = m.pair_friction[k][0];
      float t = m.body_invweight0[b1] + m.body_invweight0[b2];
      float iw = (t + mu * mu * t) * 2.f * mu * mu / m.impratio;
      float k_, b_, imp;
      kbi(m.timestep, m.pair_solref[k], m.pair_solimp[k], pos, k_, b_, imp);
      float Rr_ = fmaxf(iw * (1.f - imp) / imp, DIAL_MINVAL);
      S.e_D = 1.f / Rr_;
      S.e_aref = -b_ * ejv - k_ * imp * pos;
    }
  }
  // ---- 9. qacc_smooth and the Newton solve (mjx solver.solve), one factor/solve site ------
  if (w.midsync) cta_sync();
  const float scale = m.meaninertia * (float)(nv > 1 ? nv : 1);
  const float mywarm = isdof ? warm[d] : 0.f;
  float g = S.qfs;
#pragma unroll
  for (int a = 0; a < NR; ++a) Rr[a] = Mr[a];
#pragma unroll
  for (int q = 0; q < NL; ++q) Rc[q] = Mc[q];
  // Pass 0 (M x = qfrc_smooth, warm-start choice) is peeled off the Newton loop: the loop body that runs
  // `iterations` times (H assembly, solve, M/J products, line search, constraint update) then stays
  // below the size of the SM's instruction cache, so its second pass is served from the cache instead
  // of being streamed again (non-resident code reaches a warp at a fraction of the issue rate).  Same
  // results, bit for bit, as a single factor/solve site inside the loop.
  int it = 0;
  bool done;
  {
    float x = star_solve2<NL, NR, SH>(w, Rr, Rc, g);
    S.qas = x;
    if (SH::nedge(M) == 0 && M.nlimited == 0) { S.qacc = x; done = true; }
    else {
      float Maw, eJw, eJs;
      star_mul_MJ<NL, NR, true, true, SH>(w, Mr, Mc, mywarm, Maw, eJw);
      star_mul_MJ<NL, NR, false, true, SH>(w, Mr, Mc, S.qas, dummy, eJs);
      eJw -= S.e_aref; eJs -= S.e_aref;
      float lJw = S.l_sign * mywarm - S.l_aref;
      float gw = (Maw - S.qfs) * (mywarm - S.qas);
      float cw = ((lJw < 0.f) ? S.l_D * lJw * lJw : 0.f) + ((eJw < 0.f) ? S.e_D * eJw * eJw : 0.f);
      float Mas = S.qfs;
      float lJs = S.l_sign * S.qas - S.l_aref;
      float cs = ((lJs < 0.f) ? S.l_D * lJs * lJs : 0.f) + ((eJs < 0.f) ? S.e_D * eJs * eJs : 0.f);
      warp_sum3(gw, cw, cs);
      const bool usewarm = (0.5f * cw + 0.5f * gw) < (0.5f * cs);
      S.qacc = usewarm ? mywarm : S.qas;
      S.Ma = usewarm ? Maw : Mas;
      S.e_Jaref = usewarm ? eJw : eJs;
      S.l_Jaref = usewarm ? lJw : lJs;
      S.cost = INFINITY;
      S.prev_cost = 0.f;
      star_update_constraint<NL, NR, SH>(w, S);
      done = false;
      if (SH::iterations(M) != 1) {
        float improvement = (S.prev_cost - S.cost) / scale;
        float gradient = sqrtf(S.gradnorm2) / scale;
        done = (improvement < m.tolerance) || (gradient < m.tolerance);
      }
    }
  }
  while (!done) {
    star_build_H<NL, NR, SH>(w, S, Mr, Mc, Rr, Rc);
    float x = star_solve2<NL, NR, SH>(w, Rr, Rc, S.grad);
    S.search = -x;
    float mv, e_jv;
    star_mul_MJ<NL, NR, true, true, SH>(w, Mr, Mc, S.search, mv, e_jv);
    linesearch_core<SH>(w, S, mv, e_jv);
    ++it;
    star_update_constraint<NL, NR, SH>(w, S);
    done = it >= SH::iterations(M);
    float improvement = (S.prev_cost - S.cost) / scale;
    float gradient = sqrtf(S.gradnorm2) / scale;
    if (SH::iterations(M) != 1) done = done || (improvement < m.tolerance) || (gradient < m.tolerance);
  }
  qacc = S.qacc;
  qacc_int = qacc;
  } else {
  // ---- 8. constraint rows ----------------------------------------------------------------
  // contact Jacobian, compact along the chain of the contact body's last dof (lane = dof)
  if (isdof) {
    V3 ca_ = v3(mycdof[0], mycdof[1], mycdof[2]), cl_ = v3(mycdof[3], mycdof[4], mycdof[5]);
    int rootb = M.body_rootidx[m.dof_bodyid[d]];
    V3 rc = ld3(rcom + 3 * rootb);
    for (int c = 0; c < m.ncon; ++c) {
      const int kc = M.con_lastdof[c];
      if (!((M.dof_ancmask[kc] >> d) & 1u)) continue;
      const int k = M.con_pair[c];
      const int p_ = M.dof_nchain[kc] - w.nch;
      float e0 = 0.f, e1 = 0.f, e2 = 0.f, e3 = 0.f;
      if (cdist[c] - (m.pair_margin[k] - m.pair_gap[k]) < 0.f) {
        V3 p = ld3(cpos + 3 * c);
        V3 jp = cl_ + cross(ca_, p - rc);
        float jn = dot(ld3(cframe + 9 * c), jp), j1 = dot(ld3(cframe + 9 * c + 3), jp), j2 = dot(ld3(cframe + 9 * c + 6), jp);
        float mu0 = m.pair_friction[k][0], mu1 = m.pair_friction[k][1];
        e0 = jn + mu0 * j1; e1 = jn - mu0 * j1; e2 = jn + mu1 * j2; e3 = jn - mu1 * j2;
      }
      J[(4 * c + 0) * MC + p_] = e0; J[(4 * c + 1) * MC + p_] = e1;
      J[(4 * c + 2) * MC + p_] = e2; J[(4 * c + 3) * MC + p_] = e3;
    }
    // joint-limit row of this dof
    int lj = M.dof_limited[d];
    if (lj >= 0) {
      float qv = qpos[m.jnt_qposadr[lj]];
      float dmin = qv - m.jnt_range[lj][0], dmax = m.jnt_range[lj][1] - qv;
      float pos = fminf(dmin, dmax) - m.jnt_margin[lj];
      if (pos < 0.f) {
        float sign = dmin < dmax ? 1.f : -1.f;
        float k_, b_, imp;
        kbi(m.timestep, m.jnt_solref[lj], m.jnt_solimp[lj], pos, k_, b_, imp);
        float Rr = fmaxf(m.dof_invweight0[d] * (1.f - imp) / imp, DIAL_MINVAL);
        S.l_sign = sign;
        S.l_D = 1.f / Rr;
        S.l_aref = -b_ * (sign * myqvel) - k_ * imp * pos;
      }
    }
  }
  // contact edge rows (lane = edge)
  float ejv = mul_J(w, myqvel);
  if (lane < M.nedge) {
    int c = lane >> 2;
    int k = M.con_pair[c];
    float pos = cdist[c] - (m.pair_margin[k] - m.pair_gap[k]);
    if (pos < 0.f) {
      int b1 = m.geom_bodyid[m.pair_geom1[k]], b2 = m.geom_bodyid[m.pair_geom2[k]];
      float mu = m.pair_friction[k][0];
      float t = m.body_invweight0[b1] + m.body_invweight0[b2];
      float iw = (t + mu * mu * t) * 2.f * mu * mu / m.impratio;
      float k_, b_, imp;
      kbi(m.timestep, m.pair_solref[k], m.pair_solimp[k], pos, k_, b_, imp);
      float Rr = fmaxf(iw * (1.f - imp) / imp, DIAL_MINVAL);
      S.e_D = 1.f / Rr;
      S.e_aref = -b_ * ejv - k_ * imp * pos;
    }
  }

  // ---- 9. qacc_smooth and the Newton solve (mjx solver.solve), one factor/solve site ------
  //   pass 0: R = M, g = qfrc_smooth            -> qacc_smooth, warm-start choice, ctx init
  //   pass n: R = H(active set), g = grad        -> search = -H^-1 grad, line search
  if (w.midsync) cta_sync();
  const float scale = m.meaninertia * (float)(nv > 1 ? nv : 1);
  const float mywarm = isdof ? warm[d] : 0.f;
  float g = S.qfs;
#pragma unroll
  for (int c = 0; c < MCU; ++c) R[c] = Mrow[c];
  int phase = 0, it = 0;
  while (true) {
    float x = tree_solve<NL, NR, MCU>(w, R, g);
    if (phase == 0) {
      S.qas = x;
      if (M.nedge == 0 && M.nlimited == 0) { S.qacc = x; break; }
      // warm start: whichever of qacc_warmstart / qacc_smooth has the lower cost
      float Maw = mul_M<MCU>(w, Mrow, mywarm);
      float eJw = mul_J(w, mywarm) - S.e_aref;
      float lJw = S.l_sign * mywarm - S.l_aref;
      float gw = (Maw - S.qfs) * (mywarm - S.qas);
      float cw = ((lJw < 0.f) ? S.l_D * lJw * lJw : 0.f) + ((eJw < 0.f) ? S.e_D * eJw * eJw : 0.f);
      float Mas = S.qfs;  // M * M^-1 qfrc_smooth (MJX multiplies it out numerically; equal up to rounding)
      float eJs = mul_J(w, S.qas) - S.e_aref;
      float lJs = S.l_sign * S.qas - S.l_aref;
      float cs = ((lJs < 0.f) ? S.l_D * lJs * lJs : 0.f) + ((eJs < 0.f) ? S.e_D * eJs * eJs : 0.f);
      warp_sum3(gw, cw, cs);
      const bool usewarm = (0.5f * cw + 0.5f * gw) < (0.5f * cs);  // gauss(qacc_smooth) = 0
      S.qacc = usewarm ? mywarm : S.qas;
      S.Ma = usewarm ? Maw : Mas;
      S.e_Jaref = usewarm ? eJw : eJs;
      S.l_Jaref = usewarm ? lJw : lJs;
      S.cost = INFINITY;
      S.prev_cost = 0.f;
    } else {
      S.search = -x;
      linesearch<MCU>(w, S, Mrow);
      ++it;
    }
    update_constraint(w, S);
    // mjx `cond`: iteration budget, cost improvement, gradient norm (rescaled)
    bool done = (phase == 1) && (it >= m.iterations);
    if (m.iterations != 1 || phase == 1) {
      float improvement = (S.prev_cost - S.cost) / scale;
      float gradient = sqrtf(S.gradnorm2) / scale;
      if (m.iterations != 1) done = done || (improvement < m.tolerance) || (gradient < m.tolerance);
    }
    if (done) break;
    phase = 1;
    build_H<MCU>(w, S, Mrow, R);
    g = S.grad;
  }
  qacc = S.qacc;
  qacc_int = qacc;

  }

  // ---- 10. semi-implicit Euler -------------------------------------------------------------
  syncwarp();
  if (isdof) {
    warm[d] = qacc;
    if (integrate) qvel[d] = myqvel + m.timestep * qacc_int;
  }
  syncwarp();
  if (integrate && isbody && jid >= 0) {
    int qa = m.jnt_qposadr[jid], dd = m.jnt_dofadr[jid];
    if (jtype == JNT_FREE) {
      for (int i = 0; i < 3; ++i) qpos[qa + i] += m.timestep * qvel[dd + i];
      V3 wv = ld3(qvel + dd + 3);
      float nrm = sqrtf(dot(wv, wv));
      V3 ax = wv * (1.f / (nrm + 1e-6f * (nrm == 0.f ? 1.f : 0.f)));
      Q4 qn = qnormalize(qmul(ldq(qpos + qa + 3), axisangle(ax, m.timestep * nrm)));
      stq(qpos + qa + 3, qn);
    } else {
      qpos[qa] += m.timestep * qvel[dd];
    }
  }
  syncwarp();
}

// ---------------------------------------------------------------------------------
// rewards (computed by lane 0 from the slab; kinematics are those of the last forward
// pass, q/qvel are post-integration — the reference's staleness, SURVEY Appendix B)
// ---------------------------------------------------------------------------------
DEV float foot_step(float duty, float cadence, float amplitude, float phase, float time) {
  const float PI = 3.14159265358979f, TWO_PI = 6.28318530717959f;
  float t = time * TWO_PI * cadence + PI;
  float a = t + PI - TWO_PI * phase;
  float angle = a - floorf(a / TWO_PI) * TWO_PI - PI;
  if (duty < 1.f) angle *= 0.5f / (1.f - duty);
  float cl = fminf(fmaxf(angle, -0.5f * PI), 0.5f * PI);
  float value = duty < 1.f ? fast_cos(cl) : 0.f;   // |cl| <= pi/2
  float fin = fabsf(value) >= 1e-6f ? fabsf(value) : 0.f;
  return amplitude * fin;
}

DEV float quat_yaw(Q4 q) {
  return atan2f(-2.f * q.x * q.y + 2.f * q.w * q.z, q.x * q.x + q.w * q.w - q.z * q.z - q.y * q.y);
}

struct BaseKin { V3 pos, vb, ab; Q4 rot; };

// Brax x / xd of body `bid` in the body frame (brax.mjx.pipeline, deploy/dial_plan.py:52-59)
DEV BaseKin base_kin(WarpCtx& w, int bid) {
  const DevModel& M = *w.M;
  BaseKin r;
  r.pos = ld3(SM(xpos) + 3 * bid);
  r.rot = ldq(SM(xquat) + 4 * bid);
  V3 ang = ld3(SM(cvel) + 6 * bid), lin = ld3(SM(cvel) + 6 * bid + 3);
  V3 off = r.pos - ld3(SM(rcom) + 3 * M.body_rootidx[bid]);
  V3 vel = lin - cross(off, ang);
  Q4 qc; qc.w = r.rot.w; qc.x = -r.rot.x; qc.y = -r.rot.y; qc.z = -r.rot.z;
  r.vb = qrot(qc, vel);
  r.ab = qrot(qc, ang * (3.14159265358979f / 180.f));
  return r;
}

#ifdef DIAL_CUSTOM_REWARD_FILE
// user reward of a custom build (include/dial_custom_reward.h)
#include "../../include/dial_custom_reward.h"
#include DIAL_CUSTOM_REWARD_FILE
#endif

// Per-foot / per-contact terms of the built-in rewards, one lane each (lanes 0..3), summed into
// lane 0 by two xor-shuffles: [0] gait term (walk envs) or contact bonus (seq-jump), [1] penalty.
// The task fields (commands, gait, stage tables, user constants) come from `T`, the rest from the plan.
template <class SH = ShapeRT>
DEV void reward_partials(WarpCtx& w, const dial_task& T, int step, int stage, float& p0, float& p1) {
  const DevModel& M = *w.M;
  const dial_plan_desc& c = w.P->c;
  const dial_model_desc& m = M.m;
  const float stepf = (float)step;
  const int f = w.lane;
  const int env = SH::env_id(c);
  p0 = 0.f; p1 = 0.f;
  if (env == DIAL_ENV_GO2_WALK || env == DIAL_ENV_H1_WALK || env == DIAL_ENV_H1_LOCO) {
    if (f < SH::nfeet(c)) {
      float zt = foot_step(T.gait_duty, T.gait_cadence, T.gait_amplitude, T.gait_phase[f], stepf * c.dt);
      float z;
      if (env == DIAL_ENV_GO2_WALK) {
        int sid = c.feet_site[f], sb = m.site_bodyid[sid];
        const float* X = SM(xmat) + 9 * sb;
        z = SM(xpos)[3 * sb + 2] + X[6] * m.site_pos[sid][0] + X[7] * m.site_pos[sid][1] + X[8] * m.site_pos[sid][2];
#ifdef DIAL_TERRAIN
        if (w.ter) {   // the foot's height above the terrain beneath it
          const float fx = SM(xpos)[3 * sb] + X[0] * m.site_pos[sid][0] + X[1] * m.site_pos[sid][1] + X[2] * m.site_pos[sid][2];
          const float fy = SM(xpos)[3 * sb + 1] + X[3] * m.site_pos[sid][0] + X[4] * m.site_pos[sid][1] + X[5] * m.site_pos[sid][2];
          float sx, sy;
          z -= terrain_at(*w.ter, fx, fy, sx, sy);
        }
#endif
        float e = (zt - z) / 0.05f;
        p0 = -e * e;
      } else if (env == DIAL_ENV_H1_WALK) {
        z = fminf(SM(cdist)[2 * f], SM(cdist)[2 * f + 1]);
        p0 = -(zt - z) * (zt - z);
      } else {   // H1 loco: two capsules (4 contacts) per foot
        z = fminf(fminf(SM(cdist)[4 * f], SM(cdist)[4 * f + 1]), fminf(SM(cdist)[4 * f + 2], SM(cdist)[4 * f + 3]));
        p0 = -(zt - z) * (zt - z);
      }
    }
  } else if (env == DIAL_ENV_GO2_SEQJUMP) {
    if (f < 4) {
      const int i = f;
      float dist = SM(cdist)[i];
      bool penal = dist <= 0.001f;
      float px = SM(cpos)[3 * i], py = SM(cpos)[3 * i + 1];
      for (int j = 0; j < T.n_stage; ++j) {
        float dx = px - T.contact_targets[j][i][0], dyy = py - T.contact_targets[j][i][1];
        bool cond = dx * dx + dyy * dyy <= T.contact_radius[j][i] * T.contact_radius[j][i];
        if (cond && j == stage) p0 += fminf(fmaxf(1.f - dist, 0.f), 1.f);
        penal = penal && !cond;
      }
      p1 = penal ? 1.f : 0.f;
    }
  } else {
    return;   // Allegro / custom: nothing per foot (warp-uniform: no shuffles needed)
  }
  // lanes 0..3 -> lane 0 in the fixed order ((0+1)+(2+3)): the same sum on every lane that needs it
  p0 += shfl_xor(p0, 1); p1 += shfl_xor(p1, 1);
  p0 += shfl_xor(p0, 2); p1 += shfl_xor(p1, 2);
}

template <class SH = ShapeRT>
DEV float reward_lane0(WarpCtx& w, const dial_task& T, int step, int& stage, float part0, float part1) {
  const DevModel& M = *w.M;
  const dial_plan_desc& c = w.P->c;
  const dial_model_desc& m = M.m;
  const float stepf = (float)step;
  const int env = SH::env_id(c);
  float rew = 0.f;
#ifdef DIAL_CUSTOM_REWARD_FILE
  if (env == DIAL_ENV_CUSTOM) {
    dial_reward_ctx x;
    x.step = step; x.dt = c.dt;
    x.nq = m.nq; x.nv = m.nv; x.nu = m.nu; x.nbody = m.nbody; x.ncon = m.ncon; x.nsite = m.nsite; x.n_user = T.n_user;
    x.qpos = SM(qpos); x.qvel = SM(qvel); x.ctrl = SM(ctrl);
    x.xpos = SM(xpos); x.xquat = SM(xquat); x.xmat = SM(xmat); x.cvel = SM(cvel);
    x.subtree_com = SM(rcom); x.body_rootidx = M.body_rootidx;
    x.contact_dist = SM(cdist); x.contact_pos = SM(cpos);
    x.site_bodyid = m.site_bodyid; x.site_pos = &m.site_pos[0][0];
    x.user = T.user;
#ifdef DIAL_TERRAIN
    x.terrain = w.ter;
#else
    x.terrain = nullptr;
#endif
    return dial_custom_reward(&x);
  }
#endif
  Q4 rot0 = ldq(SM(xquat) + 4);  // x.rot[0]
  V3 up = qrot(rot0, v3(0, 0, 1));
  float r_upright = -(up.x * up.x + up.y * up.y + (up.z - 1.f) * (up.z - 1.f));
  BaseKin bk = base_kin(w, c.torso_body);
  if (env == DIAL_ENV_ALLEGRO) {
    // manipulation.py:75-84: ball angular velocity / position tracking + joint deviation
    const int ob = c.torso_body;
    V3 wv = ld3(SM(cvel) + 6 * ob) * (3.14159265358979f / 180.f);
    V3 dw = wv - ld3(T.ang_cmd);
    V3 dp = ld3(SM(xpos) + 3 * ob) - ld3(T.pos_tar);
    float rj = 0.f;
    for (int a = 0; a < SH::nu(M); ++a) { float e = SM(qpos)[7 + a] - c.joint_offset[a]; rj -= e * e; }
    return -dot(dw, dw) - 5.f * dot(dp, dp) + 0.1f * rj;
  }
  if (env == DIAL_ENV_GO2_WALK || env == DIAL_ENV_H1_WALK || env == DIAL_ENV_H1_LOCO) {
    float ramp = stepf * c.dt / c.ramp_up_time;
    // randomize_tasks: a one-step command override (dial_plan_set_command / the task's cmd_step)
    const float* vel_cmd = step == T.cmd_step ? T.cmd_vel : T.vel_cmd;
    const float* ang_cmd = step == T.cmd_step ? T.cmd_ang : T.ang_cmd;
    float vtx = fminf(vel_cmd[0] * ramp, vel_cmd[0]), vty = fminf(vel_cmd[1] * ramp, vel_cmd[1]);
    float atz = fminf(ang_cmd[2] * ramp, ang_cmd[2]);
    const float r_gaits = part0;   // per-foot terms: reward_partials
    float yaw_tar = 0.f + atz * c.dt * stepf;
    float dyaw = quat_yaw(bk.rot) - yaw_tar;
    // atan2(sin d, cos d) == d wrapped to (-pi, pi]
    float wy = dyaw - 6.28318530717959f * rintf(dyaw * 0.159154943091895f);
    float r_yaw = -wy * wy;
    float r_vel = -((bk.vb.x - vtx) * (bk.vb.x - vtx) + (bk.vb.y - vty) * (bk.vb.y - vty));
    float r_ang = -(bk.ab.z - atz) * (bk.ab.z - atz);
    float bz = bk.pos.z;
#ifdef DIAL_TERRAIN
    if (w.ter) { float sx, sy; bz -= terrain_at(*w.ter, bk.pos.x, bk.pos.y, sx, sy); }   // above the terrain beneath
#endif
    float r_h = -(bz - T.pos_tar[2]) * (bz - T.pos_tar[2]);
    if (env == DIAL_ENV_GO2_WALK) {
      rew = 0.1f * r_gaits + 0.5f * r_upright + 0.3f * r_yaw + r_vel + r_ang + r_h;
    } else if (env == DIAL_ENV_H1_LOCO) {
      // unitree_h1_env.py:774-800: all three body-rate components, foot-level and energy terms
      float atx = fminf(ang_cmd[0] * ramp, ang_cmd[0]), aty = fminf(ang_cmd[1] * ramp, ang_cmd[1]);
      float r_ang3 = -((bk.ab.x - atx) * (bk.ab.x - atx) + (bk.ab.y - aty) * (bk.ab.y - aty) + (bk.ab.z - atz) * (bk.ab.z - atz));
      float r_level = 0.f;
      for (int f = 0; f < SH::nfeet(c); ++f) {
        const float* X = SM(xmat) + 9 * m.site_bodyid[c.feet_site[f]];
        r_level -= X[2] * X[2] + X[5] * X[5] + (X[8] - 1.f) * (X[8] - 1.f);
      }
      float r_energy = 0.f;
      for (int a = 0; a < SH::nu(M); ++a) { float e = SM(ctrl)[a] / c.joint_torque_range[a][1] * SM(qvel)[6 + a] / 160.f; r_energy -= e * e; }
      rew = 10.f * r_gaits + 0.5f * r_upright + 0.5f * r_yaw + r_vel + r_ang3 + 0.5f * r_h + 0.02f * r_level + 0.01f * r_energy;
    } else {
      float r_energy = 0.f;
      for (int a = 0; a < SH::nu(M); ++a) { float e = SM(ctrl)[a] / c.joint_torque_range[a][1]; r_energy -= e * e; }
      rew = 5.f * r_gaits + 0.5f * r_upright + 0.1f * r_yaw + r_vel + r_ang + 0.5f * r_h + 0.01f * r_energy;
    }
  } else {  // DIAL_ENV_GO2_SEQJUMP
    V3 dp = bk.pos - ld3(T.pose_seq[stage]);
    float r_pos = -dot(dp, dp);
    float dy = quat_yaw(bk.rot) - T.yaw_seq[stage];
    float r_yaw = -dy * dy;
    const float r_contact = part0, pen = part1;   // per-contact terms: reward_partials
    rew = r_pos + r_upright + 0.3f * r_yaw + 0.1f * r_contact - 0.1f * pen + 10.f;
    // IEEE division: -use_fast_math would make it a * (1 / b), whose floor differs from the host's at boundaries
    // of jump_dt that are not powers of two (the host, the C port and the reference divide in fp32)
    int ns = (int)floorf(__fdiv_rn((float)(step + 1) * c.dt, T.jump_dt));
    stage = ns < T.n_stage - 1 ? ns : T.n_stage - 1;
  }
  return rew;
}

// ---------------------------------------------------------------------------------
// the per-warp rollout: one sample row, H env steps
// ---------------------------------------------------------------------------------
template <int NL, int NR, class SH = ShapeRT>
DEV void rollout_warp(const DevModel* Mp, const DevPlan* Pp, float* slab, const RolloutArgs& A,
                      int row, int lane) {
  WarpCtx w;
  w.M = Mp; w.P = Pp; w.s = slab; w.lane = lane;
  w.midsync = A.lockstep >= 2;
  w.itersync = A.lockstep >= 3;
  w.dbg = A.dbg;
  const DevModel& M = *Mp;
  const dial_model_desc& m = M.m;
  const dial_plan_desc& c = Pp->c;
  const int nq = SH::nq(M), nv = SH::nv(M), nu = SH::nu(M), nb = SH::nbody(M);
  // instance of a batched launch and the row inside it (the sample index)
  const int inst = A.rows_per_inst > 0 ? row / A.rows_per_inst : 0;
  const int lrow = row - inst * A.rows_per_inst;
#ifdef DIAL_TERRAIN
  w.ter = A.terrain && A.terrain[inst].nx > 0 ? A.terrain + inst : nullptr;
#endif
  // ancestor chain of this lane's dof
  w.nch = 0; w.ndesc = 0; w.mylevel = -1; w.parent = -1;
#pragma unroll
  for (int i = 0; i < DIAL_MAXCHAIN; ++i) w.chain[i] = 0;
  if (lane < nv) {
    w.nch = M.dof_nchain[lane];
    w.ndesc = M.dof_ndesc[lane];
    w.mylevel = M.dof_level[lane];
    w.parent = m.dof_parentid[lane];
#pragma unroll
    for (int i = 0; i < DIAL_MAXCHAIN; ++i)
      if (i < w.nch) w.chain[i] = M.chain_tab[lane][i];
  }
  // star layout: lane constants, and the scratch zeroed once (padding slots are never written again)
  w.s_pos = 0; w.s_col = 0; w.s_cb = 0; w.s_chain = -2; w.s_depth = 0; w.s_top = 0; w.s_conmask = 0u; w.e_cb = 0;
  if constexpr (NL > 0) {
    using SD = StarDims<NL, NR>;
    w.s_cb = SD::NRP; w.e_cb = SD::NRP;
    if (lane < nv) {
      w.s_pos = M.s_pos[lane]; w.s_chain = M.s_chain[lane]; w.s_depth = M.s_depth[lane];
      if (w.s_chain >= 0) { w.s_cb = SD::NRP + w.s_chain * SD::CS; w.s_col = SD::NRP + w.s_depth; w.s_top = M.s_top[w.s_chain]; }
      else w.s_col = w.s_depth;
      for (int c = 0; c < SH::ncon(M); ++c)
        if (w.s_chain < 0 || M.s_con_chain[c] == w.s_chain) w.s_conmask |= 1u << c;
    }
    if (lane < SH::nedge(M)) { const int cc = M.s_con_chain[lane >> 2]; if (cc >= 0) w.e_cb = SD::NRP + cc * SD::CS; }
    const int nz = 2 * M.s_npos * SD::RS + SH::nedge(M) * SD::RS + M.s_npos + 8;   // Ms, Hs, Js, xs are contiguous
    for (int i = lane; i < nz; i += 32) SM(Ms)[i] = 0.f;
    for (int i = lane; i < 32; i += 32) SM(frow)[i] = 0.f;
  }
  // initial state + world body constants
  for (int i = lane; i < nq; i += 32) SM(qpos)[i] = A.qpos0[(size_t)inst * nq + i];
  for (int i = lane; i < nv; i += 32) { SM(qvel)[i] = A.qvel0[(size_t)inst * nv + i]; SM(warm)[i] = A.warm0[(size_t)inst * nv + i]; }
  if (lane == 0) {
    SM(xpos)[0] = SM(xpos)[1] = SM(xpos)[2] = 0.f;
    SM(xquat)[0] = 1.f; SM(xquat)[1] = SM(xquat)[2] = SM(xquat)[3] = 0.f;
    for (int i = 0; i < 9; ++i) SM(xmat)[i] = (i % 4 == 0) ? 1.f : 0.f;
    for (int i = 0; i < 3; ++i) SM(xipos)[i] = 0.f;
    for (int i = 0; i < 10; ++i) SM(cinert)[i] = 0.f;
    for (int i = 0; i < 6; ++i) { SM(cvel)[i] = 0.f; SM(cfrc)[i] = 0.f; }
    SM(cacc)[0] = SM(cacc)[1] = SM(cacc)[2] = 0.f;
    SM(cacc)[3] = -m.gravity[0]; SM(cacc)[4] = -m.gravity[1]; SM(cacc)[5] = -m.gravity[2];
  }
  syncwarp();

  // control knots of this sample (lane = actuator)
  const int Hn1 = c.Hnode + 1;
  float Y[DIAL_MAXNODE];
#pragma unroll
  for (int k = 0; k < DIAL_MAXNODE; ++k) Y[k] = 0.f;
  if (A.mode == 1 && lane < nu) {
    // the sample index: every member of an ensemble rolls the same samples
    const int smp = A.rows_per_model > 0 ? lrow % A.rows_per_model : lrow;
    const bool is_mean = smp == c.Nsample;
    const uint32_t gidx = (uint32_t)(c.shard_offset + smp);
    const uint32_t ntot = (uint32_t)c.Ntotal * (uint32_t)Hn1 * (uint32_t)nu;
    uint32_t key0 = A.key_dev ? A.key_dev[2 * inst] : A.key0, key1 = A.key_dev ? A.key_dev[2 * inst + 1] : A.key1;
    if (A.rng_dev) split_key(A.rng_dev[2 * inst], A.rng_dev[2 * inst + 1], key0, key1);
    const float* noise = schedule_noise(A.sched, inst, A.iter, A.noise);
#pragma unroll
    for (int k = 0; k < DIAL_MAXNODE; ++k) {
      if (k < Hn1) {
        float yb = A.Ybar[(inst * Hn1 + k) * nu + lane];
        float y = yb;
        if (!is_mean && k > 0) {
          uint32_t idx = (gidx * (uint32_t)Hn1 + (uint32_t)k) * (uint32_t)nu + (uint32_t)lane;
          float e = A.eps ? A.eps[idx] : jax_normal_legacy(key0, key1, idx, ntot);
          y = e * noise[k] + yb;
        }
        Y[k] = fminf(fmaxf(y, -1.f), 1.f);
      }
    }
  }

  int step = A.counters_in ? A.counters_in[2 * inst] : A.step0, stage = A.counters_in ? A.counters_in[2 * inst + 1] : A.stage0;
  float rsum = 0.f;
  const bool fwd_only = A.mode == 2;  // pipeline_init: mjx.forward only, zero ctrl
  const int H = fwd_only ? 1 : A.H;
  const int nfr = fwd_only ? 1 : SH::n_frames(c);
  for (int t = 0; t < H; ++t) {
    if (A.lockstep && (A.sync_every <= 1 || t % A.sync_every == 0)) cta_sync();
    // action -> joint target -> torque (base_env.py:37-66)
    if (lane < nu && fwd_only) SM(ctrl)[lane] = 0.f;
    if (lane < nu && !fwd_only) {
      float u;
      if (A.mode == 0) {
        u = A.us[(size_t)row * (A.us_row ? A.us_row : A.H * nu) + t * nu + lane];
      } else {
        u = 0.f;
#pragma unroll
        for (int k = 0; k < DIAL_MAXNODE; ++k)
          if (k < Hn1) u += c.M_n2u[t][k] * Y[k];
      }
      float an = (u * c.action_scale + 1.f) * 0.5f;
      float jt = c.joint_range[lane][0] + c.joint_offset[lane] + an * (c.joint_range[lane][1] - c.joint_range[lane][0]);
      jt = fminf(fmaxf(jt, c.physical_joint_range[lane][0]), c.physical_joint_range[lane][1]);
      float ctrl = jt;
      if (c.leg_control_torque) {
        float tau = c.kp[lane] * (jt - SM(qpos)[7 + lane]) - c.kd[lane] * SM(qvel)[6 + lane];
        ctrl = fminf(fmaxf(tau, c.joint_torque_range[lane][0]), c.joint_torque_range[lane][1]);
      }
      SM(ctrl)[lane] = ctrl;
    }
    syncwarp();
    for (int f = 0; f < nfr; ++f) physics_step<NL, NR, SH>(w, !fwd_only);
    if (fwd_only) break;
    float rew = 0.f, part0, part1;
    // the task of this row, derived here from `row` (live anyway) and the launch arguments so that no
    // register holds it over the physics step
    const dial_task& T = A.tasks ? A.tasks[A.task_rows > 0 ? row / A.task_rows : 0] : plan_task(c);
    reward_partials<SH>(w, T, step, stage, part0, part1);
    if (lane == 0) rew = reward_lane0<SH>(w, T, step, stage, part0, part1);
    stage = shfl_i(stage, 0);
    step += 1;
    rsum += rew;
    // per-step outputs (coalesced: consecutive lanes -> consecutive addresses)
    size_t rt = (size_t)row * A.H + t;
    if (A.rewss && lane == 0) A.rewss[rt] = rew;
    if (A.q) for (int i = lane; i < nq; i += 32) A.q[rt * nq + i] = SM(qpos)[i];
    if (A.qd) for (int i = lane; i < nv; i += 32) A.qd[rt * nv + i] = SM(qvel)[i];
    if (A.xpos) for (int i = lane; i < 3 * (nb - 1); i += 32) A.xpos[rt * 3 * (nb - 1) + i] = SM(xpos)[3 + i];
  }
  if (A.rews && lane == 0 && !fwd_only) A.rews[row] = rsum / (float)A.H;
#ifndef DIAL_NO_XCH
  if (A.xch_world > 1 && lane == 0 && !fwd_only && A.mode == 1) {
    // sample rows go to every rank's mailbox at their GLOBAL index; the mean row (rolled by every
    // rank, bitwise identical) only to the local one
    const float val = rsum / (float)A.H;
    const uint32_t buf = (*A.xch_seq) & 1u;
    const size_t base = (size_t)buf * (size_t)(c.Ntotal + 1);
    const bool sample = row < c.Nsample;
    const size_t slot = base + (size_t)(sample ? c.shard_offset + row : c.Ntotal);
    for (int p = 0; p < A.xch_world; ++p)
      if (sample || p == A.xch_rank) A.xch_mbox[p][slot] = val;
  }
#endif
  // final state of each instance's first row.  The instance is derived again from a shuffled copy of
  // `row`, which the compiler cannot equate with the prologue's: inst / lrow are not kept live over
  // the env-step loop (two registers the star kernels do not have to spare).
  const int erow = shfl_i(row, 0), einst = A.rows_per_inst > 0 ? erow / A.rows_per_inst : 0;
  if (erow == einst * A.rows_per_inst) {
    const int inst = einst;
    if (A.qpos_out) for (int i = lane; i < nq; i += 32) A.qpos_out[(size_t)inst * nq + i] = SM(qpos)[i];
    if (A.qvel_out) for (int i = lane; i < nv; i += 32) A.qvel_out[(size_t)inst * nv + i] = SM(qvel)[i];
    if (A.warm_out) for (int i = lane; i < nv; i += 32) A.warm_out[(size_t)inst * nv + i] = SM(warm)[i];
    if (A.ctrl_out) for (int i = lane; i < nu; i += 32) A.ctrl_out[(size_t)inst * nu + i] = SM(ctrl)[i];
    if (A.kin_out && lane == 0) {   // what the envs' _get_obs reads of pipeline_state.x / xd (kinematics of the last forward pass)
      const BaseKin bk = base_kin(w, c.torso_body);
      float* ko = A.kin_out + 13 * inst;
      ko[0] = bk.pos.x; ko[1] = bk.pos.y; ko[2] = bk.pos.z;
      ko[3] = bk.rot.w; ko[4] = bk.rot.x; ko[5] = bk.rot.y; ko[6] = bk.rot.z;
      ko[7] = bk.vb.x; ko[8] = bk.vb.y; ko[9] = bk.vb.z;
      ko[10] = bk.ab.x; ko[11] = bk.ab.y; ko[12] = bk.ab.z;
    }
    if (A.counters_out && lane == 0) { A.counters_out[2 * inst] = step; A.counters_out[2 * inst + 1] = stage; }
  }
}
