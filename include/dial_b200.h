/*
 * dial_b200.h — C ABI of the H100-native DIAL-MPC sampling core.
 *
 * The reference (LeCAR-Lab/dial-mpc) has no FFI for this path: its boundary is the
 * Python class `MBDPI` plus the env registry, and every function below replaces a
 * piece of jitted JAX that `MBDPI` calls.  Each entry point cites the reference
 * code it stands in for (paths relative to the reference root).
 *
 * Conventions
 *   - extern "C", opaque handles, plain pointers and sizes, no torch / C++ types.
 *   - every `const float* / float*` argument marked [dev] is a CUDA device pointer to
 *     contiguous row-major fp32 owned by the caller; `stream` is a `cudaStream_t`
 *     passed as `void*`; all work is enqueued asynchronously on it.
 *   - return 0 on success, negative on error; `dial_last_error()` returns a static,
 *     thread-local, NUL-terminated description of the last failure.
 *   - one plan per GPU; a plan is not thread-safe.
 *   - no hidden allocations after `dial_plan_create`.
 */
#ifndef DIAL_B200_H_
#define DIAL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DIAL_ABI_VERSION 14

/* capacities of the fixed-size device model */
#define DIAL_MAXB 24   /* bodies incl. world            */
#define DIAL_MAXV 28   /* dofs                          */
#define DIAL_MAXQ 29   /* generalized positions         */
#define DIAL_MAXU 20   /* actuators                     */
#define DIAL_MAXG 8    /* collision geoms               */
#define DIAL_MAXP 16   /* contact pairs                 */
#define DIAL_MAXC 20   /* contacts                      */
#define DIAL_MAXS 8    /* sites                         */
#define DIAL_MAXNODE 8 /* Hnode+1                       */
#define DIAL_MAXH 64   /* Hsample+1                     */
#define DIAL_MAXSTAGE 12
#define DIAL_MAXUSER 64 /* user constants of a custom reward */
#define DIAL_MAXRANK 8  /* GPUs of one NVLink domain sharing the samples */
#define DIAL_MAXENS 16  /* planning models (ensemble members) of one instance */
#define DIAL_MAXDIFFUSE 64 /* diffusion iterations of one control step (dial_mpc_step) */
#define DIAL_MAXDELAY 16   /* control steps of latency of one instance (dial_plan_set_instance_delay) */
#define DIAL_MAXPUSH 16    /* entries of one instance's push table (dial_plan_set_instance_pushes) */
#define DIAL_MAXSUBSTEPS 16 /* physics substeps per plan physics step of one instance's plant (dial_plan_set_instance_plant) */
#define DIAL_MAXTERRAIN 1024 /* grid vertices per side of one instance's terrain (dial_plan_set_instance_terrain) */
#define DIAL_TERRAIN_PLANT 0   /* the side of dial_plan_set_instance_terrain: the plant's env step */
#define DIAL_TERRAIN_PLANNER 1 /* the planner's rollouts, ensemble members, adaptation and predictions */
#define DIAL_IPC_HANDLE_BYTES 64

/* environments (reward functors fused into the rollout kernel) */
enum {
  DIAL_ENV_GO2_WALK = 0,    /* UnitreeGo2Env.step         envs/unitree_go2_env.py:126-261 */
  DIAL_ENV_GO2_SEQJUMP = 1, /* UnitreeGo2SeqJumpEnv.step  envs/unitree_go2_env.py:403-521 */
  DIAL_ENV_H1_WALK = 2,     /* UnitreeH1WalkEnv.step      envs/unitree_h1_env.py:181-321  */
  DIAL_ENV_ALLEGRO = 3,     /* AllegroReorientEnv.step    envs/manipulation.py:63-100     */
  DIAL_ENV_H1_LOCO = 4,     /* UnitreeH1LocoEnv.step      envs/unitree_h1_env.py:686-830  */
  DIAL_ENV_CUSTOM = 5,      /* user reward (README.md:223-312 "Writing Custom Environment"):
                               a device functor compiled into a dedicated build of this library,
                               see include/dial_custom_reward.h                              */
};

/* Compiled robot model: what `brax.io.mjcf.load` + `mjx.put_model` give the reference
 * (envs/unitree_go2_env.py:95-99).  Filled by the host-side model compiler. */
typedef struct dial_model_desc {
  int32_t nq, nv, nu, nbody, njnt, ngeom, nsite, npair, ncon;
  int32_t iterations, ls_iterations, eulerdamp, cone;
  float timestep, gravity[3], tolerance, ls_tolerance, impratio, meaninertia;
  /* bodies (index 0 = world) */
  int32_t body_parentid[DIAL_MAXB], body_rootid[DIAL_MAXB], body_depth[DIAL_MAXB];
  int32_t body_jntadr[DIAL_MAXB], body_dofadr[DIAL_MAXB], body_dofnum[DIAL_MAXB];
  float body_pos[DIAL_MAXB][3], body_quat[DIAL_MAXB][4];
  float body_ipos[DIAL_MAXB][3], body_iquat[DIAL_MAXB][4];
  float body_mass[DIAL_MAXB], body_inertia[DIAL_MAXB][3], body_invweight0[DIAL_MAXB];
  float body_invweight0_rot[DIAL_MAXB];
  /* joints (at most one per body) */
  int32_t jnt_type[DIAL_MAXB], jnt_qposadr[DIAL_MAXB], jnt_dofadr[DIAL_MAXB], jnt_limited[DIAL_MAXB];
  float jnt_pos[DIAL_MAXB][3], jnt_axis[DIAL_MAXB][3], jnt_range[DIAL_MAXB][2], jnt_margin[DIAL_MAXB];
  float jnt_solref[DIAL_MAXB][2], jnt_solimp[DIAL_MAXB][5];
  /* dofs */
  int32_t dof_bodyid[DIAL_MAXV], dof_jntid[DIAL_MAXV], dof_parentid[DIAL_MAXV];
  float dof_armature[DIAL_MAXV], dof_damping[DIAL_MAXV], dof_invweight0[DIAL_MAXV];
  float qpos0[DIAL_MAXQ];
  /* collision geoms + static contact pairs (MJX fixed-size contact arrays) */
  int32_t geom_type[DIAL_MAXG], geom_bodyid[DIAL_MAXG];
  float geom_pos[DIAL_MAXG][3], geom_quat[DIAL_MAXG][4], geom_size[DIAL_MAXG][3];
  int32_t pair_kind[DIAL_MAXP], pair_geom1[DIAL_MAXP], pair_geom2[DIAL_MAXP], pair_ncon[DIAL_MAXP];
  int32_t pair_condim[DIAL_MAXP];
  float pair_friction[DIAL_MAXP][5], pair_margin[DIAL_MAXP], pair_gap[DIAL_MAXP];
  float pair_solref[DIAL_MAXP][2], pair_solimp[DIAL_MAXP][5];
  /* sites */
  int32_t site_bodyid[DIAL_MAXS];
  float site_pos[DIAL_MAXS][3];
  /* actuators (joint transmissions): force = gain*ctrl + b0 + b1*q + b2*qd */
  int32_t actuator_dofadr[DIAL_MAXU], actuator_qposadr[DIAL_MAXU];
  int32_t actuator_ctrllimited[DIAL_MAXU], actuator_forcelimited[DIAL_MAXU];
  float actuator_gear[DIAL_MAXU], actuator_gain[DIAL_MAXU], actuator_bias[DIAL_MAXU][3];
  float actuator_ctrlrange[DIAL_MAXU][2], actuator_forcerange[DIAL_MAXU][2];
} dial_model_desc;

/* Environment + planner configuration: DialConfig (core/dial_config.py:4-23),
 * BaseEnvConfig (config/base_env_config.py:4-20) and the env-specific constants. */
typedef struct dial_plan_desc {
  int32_t env_id;
  int32_t Nsample;   /* samples rolled by THIS rank (shard size)                  */
  int32_t Ntotal;    /* Nsample of the whole job (== Nsample when not sharded)    */
  int32_t shard_offset; /* global index of this rank's first sample               */
  int32_t Hsample, Hnode;
  int32_t n_frames;  /* int(dt / timestep), base_env.py:17                        */
  int32_t leg_control_torque; /* 1: act2tau, 0: act2joint -> position actuator    */
  float temp_sample;
  float dt, action_scale;
  float kp[DIAL_MAXU], kd[DIAL_MAXU];
  float joint_range[DIAL_MAXU][2];          /* env.joint_range (sampling range)   */
  float physical_joint_range[DIAL_MAXU][2]; /* sys.jnt_range[1:]                  */
  float joint_torque_range[DIAL_MAXU][2];   /* sys.actuator_ctrlrange (+-inf ok)  */
  float joint_offset[DIAL_MAXU];            /* added to the joint target (Allegro: init_q[7:], manipulation.py:106) */
  float M_n2u[DIAL_MAXH][DIAL_MAXNODE];     /* node -> action spline matrix       */
  /* reward constants */
  int32_t torso_body;       /* MuJoCo body id of the torso (x index + 1)          */
  int32_t nfeet;
  int32_t feet_site[4];
  float ramp_up_time;
  /* ---- the task: vel_cmd .. user is laid out exactly as dial_task below (the kernels read a plan's
   * own task through a dial_task view of this block) ---- */
  float vel_cmd[3], ang_cmd[3], pos_tar[3];
  float gait_duty, gait_cadence, gait_amplitude, gait_phase[4];
  /* randomize_tasks (unitree_go2_env.py:141-155, unitree_h1_env.py:198-212): the env step whose
   * info["step"] equals cmd_step uses (cmd_vel, cmd_ang) instead of (vel_cmd, ang_cmd); -1 = none.
   * Set through dial_plan_set_command only (dial_plan_create ignores the value and starts at -1). */
  int32_t cmd_step;
  float cmd_vel[3], cmd_ang[3];
  /* seq-jump */
  int32_t n_stage;
  float jump_dt;
  float pose_seq[DIAL_MAXSTAGE][3], yaw_seq[DIAL_MAXSTAGE];
  float contact_targets[DIAL_MAXSTAGE][4][3], contact_radius[DIAL_MAXSTAGE][4];
  /* DIAL_ENV_CUSTOM: constants handed to dial_custom_reward() (ctx->user) */
  int32_t n_user;
  float user[DIAL_MAXUSER];
  /* ---- end of the task ---- */
  /* independent planner instances of one plan (0 or 1: a single instance).  B > 1 instances share
   * the model, every constant above and the annealing schedule; each has its own state, counters,
   * rng, control knots and outputs (see dial_mpc_buffers).  Batched plans run through dial_mpc_step
   * only, with the fused update; they cannot be sharded (Ntotal == Nsample) and need
   * Nsample + 1 <= 2^17. */
  int32_t n_inst;
  /* ensemble planning (0..DIAL_MAXENS).  0: every rollout row of instance b runs instance b's model (the
   * default).  K >= 1: instance b plans against K member models (dial_plan_set_ensemble_model) while its
   * env step runs its instance model (dial_plan_set_instance_model), the plant.  Each reverse_once of
   * dial_mpc_step rolls all Nsample+1 rows of instance b once per member, with the same perturbations,
   * and scores sample i by a risk measure of its K rewards: the fp32 mean (summed in member order, then
   * divided by K) unless dial_plan_set_ensemble_risk chose CVaR or the worst case for instance b.
   * Sharded plans reject n_ens >= 1. */
  int32_t n_ens;
} dial_plan_desc;

/* The task of one planner instance: exactly the reward inputs that differ between tasks of one model,
 * with the names, meanings and layout of the dial_plan_desc block vel_cmd .. user above.  Everything else (model, gains, joint
 * ranges, dt, ramp_up_time, torso body, feet sites, Nsample, annealing schedule) stays in the plan.
 * The kernels trust the counts: a task must hold 1 <= n_stage <= DIAL_MAXSTAGE and
 * 0 <= n_user <= DIAL_MAXUSER (dial_plan_get_task and the Python helpers check this; a caller that
 * writes tasks itself must too). */
typedef struct dial_task {
  float vel_cmd[3], ang_cmd[3], pos_tar[3];
  float gait_duty, gait_cadence, gait_amplitude, gait_phase[4];
  int32_t cmd_step;                 /* randomize_tasks one-step command; -1 = none */
  float cmd_vel[3], cmd_ang[3];
  int32_t n_stage;                  /* 1..DIAL_MAXSTAGE */
  float jump_dt;
  float pose_seq[DIAL_MAXSTAGE][3], yaw_seq[DIAL_MAXSTAGE];
  float contact_targets[DIAL_MAXSTAGE][4][3], contact_radius[DIAL_MAXSTAGE][4];
  int32_t n_user;
  float user[DIAL_MAXUSER];
} dial_task;

/* State handed to the planner: Brax `State.pipeline_state` (qpos, qvel,
 * qacc_warmstart) + `State.info` counters the rewards read
 * (envs/unitree_go2_env.py:106-118, :366-381). */
typedef struct dial_state {
  const float* qpos;           /* [dev] [nq] */
  const float* qvel;           /* [dev] [nv] */
  const float* qacc_warmstart; /* [dev] [nv] */
  int32_t step;                /* info["step"]          */
  int32_t stage;               /* info["contact_stage"] */
} dial_state;

typedef struct dial_plan dial_plan;

int dial_abi_version(void);
const char* dial_last_error(void);
/* sizeof() of the descriptor structs as compiled into the library: which = 0 model, 1 plan,
 * 2 state, 3 mpc buffers, 4 task, 5 push, 6 plant, 7 terrain (lets foreign-language bindings verify their struct
 * layout). */
size_t dial_sizeof(int which);

/* Create / destroy a plan (uploads model + config, allocates all workspaces). */
dial_plan* dial_plan_create(const dial_model_desc* model, const dial_plan_desc* cfg);
void dial_plan_destroy(dial_plan* plan);

/* rollout_us_vmap — core/dial_core.py:36-42,80-81: roll B action sequences from one
 * state.  us [dev] [B, Hsample+1, nu]; outputs (nullable except rewss):
 * rewss [B,Hs+1], q [B,Hs+1,nq], qd [B,Hs+1,nv], xpos [B,Hs+1,nbody-1,3]. */
int dial_rollout(dial_plan* plan, const dial_state* s, const float* us, int B, int H,
                 float* rewss, float* q, float* qd, float* xpos, void* stream);

/* env.step for ONE instance — the `step_env(state, Y0[0])` call at
 * core/dial_core.py:245.  Writes the successor state (qpos,qvel,qacc_warmstart
 * [dev]), the reward [dev][1] and ctrl [dev][nu]; step/stage are advanced by the host. */
int dial_env_step(dial_plan* plan, const dial_state* s, const float* action,
                  float* qpos_out, float* qvel_out, float* warm_out, float* reward,
                  float* ctrl_out, void* stream);

/* randomize_tasks support: replaces the command of ONE env step (the one whose info["step"]
 * == cmd_step; pass -1 for none) in every later launch of this plan — the reference draws a
 * one-step random command whenever step % 500 == 0 (unitree_go2_env.py:141-163), from a key chain
 * that depends only on the reset key, so the host can compute it ahead of the horizon reaching it.
 * Stream-ordered (safe between replays of the control-step graph). */
int dial_plan_set_command(dial_plan* plan, int cmd_step, const float vel[3], const float ang[3], void* stream);

/* randomize_tasks of UnitreeGo2SeqJumpEnv (unitree_go2_env.py:383-394, 594-631): `reset` draws a
 * whole jump sequence (11 stages) instead of using the configured one.  Replaces the stage tables
 * of the plan (n_stage <= DIAL_MAXSTAGE; pose [n][3], yaw [n], contact_targets [n][4][3],
 * contact_radius [n][4], host pointers) for every later launch.  Stream-ordered like
 * dial_plan_set_command. */
int dial_plan_set_stages(dial_plan* plan, int n_stage, const float* pose_seq, const float* yaw_seq,
                         const float* contact_targets, const float* contact_radius, void* stream);

/* The plan's current task (its dial_plan_desc reward inputs, including what dial_plan_set_command /
 * _set_stages last put there) as a dial_task [host]: a starting point for per-instance tasks
 * (dial_mpc_buffers.tasks).  Fails if the plan's counts are out of range. */
int dial_plan_get_task(const dial_plan* plan, dial_task* out);

/* The same step, also returning what the envs' `_get_obs` (envs/unitree_go2_env.py:263-286,
 * unitree_h1_env.py:323-346) reads of pipeline_state.x / xd: kin_out [dev][13] = x.pos(3),
 * x.rot(4) of the torso body, then global_to_body_velocity(xd.vel) (3) and
 * global_to_body_velocity(xd.ang * pi/180) (3) (nullable). */
int dial_env_step_kin(dial_plan* plan, const dial_state* s, const float* action,
                      float* qpos_out, float* qvel_out, float* warm_out, float* reward,
                      float* ctrl_out, float* kin_out, void* stream);

/* pipeline_init — envs/unitree_go2_env.py:104: mjx.forward at (qpos, qvel=0):
 * normalises the quaternion and produces the initial qacc_warmstart. */
int dial_pipeline_init(dial_plan* plan, const float* qpos, const float* qvel,
                       float* qpos_out, float* warm_out, void* stream);

/* Stage 1 of MBDPI.reverse_once (core/dial_core.py:103-125): sample Y0s
 * (eps injected [dev][Ntotal,Hnode+1,nu], or NULL -> Threefry stream keyed by
 * `key`), pin node 0, append the mean row, clip, spline to actions, roll out
 * this rank's shard + the mean sample and write per-sample mean rewards
 * rews_local [dev][Nsample+1] (mean sample last).  Trajectories
 * (q/qd/xpos [Nsample+1,Hs+1,*]) are kept in the plan's workspace, which is double-buffered:
 * dial_reverse_trajbar enqueued (on any stream, after the matching update) before the NEXT
 * dial_reverse_rollout reads the buffer of this rollout, so it may overlap the next rollout;
 * the buffer is reused by the rollout after next. */
int dial_reverse_rollout(dial_plan* plan, const dial_state* s, const float* eps,
                         const uint32_t key[2], const float* Ybar /*[dev][Hn+1,nu]*/,
                         const float* noise_scale /*[dev][Hn+1]*/, float* rews_local,
                         void* stream);

/* Stage 2 (core/dial_core.py:126-135): population std, softmax weights over the
 * Ntotal+1 rewards rews_all [dev] (sample-major, mean sample last) and the weighted
 * control update Ybar_out [dev][Hn+1,nu].  Every rank recomputes all Y0s from
 * eps/key, so sharded runs need only the one allgather of rewards.  Optional
 * (nullable) weights [dev][Ntotal+1]. */
int dial_reverse_update(dial_plan* plan, const float* eps, const uint32_t key[2],
                        const float* Ybar, const float* noise_scale, const float* rews_all,
                        float* Ybar_out, float* weights, void* stream);

/* dial_reverse_update with the rewards taken from this rank's exchange mailbox when
 * rews_all == NULL (see dial_exchange_*); rews_gathered (nullable) [dev][Ntotal+1] receives a
 * compact copy of the gathered rewards (the `rews` of the reference's info dict). */
int dial_reverse_update_x(dial_plan* plan, const float* eps, const uint32_t key[2],
                          const float* Ybar, const float* noise_scale, const float* rews_all,
                          float* Ybar_out, float* weights, float* rews_gathered, void* stream);

/* Stage 2 as the control-step graph runs it (dial_mpc_step): ONE launch of the fused update kernel
 * (statistics, softmax, Ybar = sum_n w_n Y0s_n with Y0s regenerated from the Threefry stream keyed
 * by split(rng)[1], rng advance) on caller buffers, for every instance of the plan (B = n_inst,
 * 1 for a single-instance plan).  All [dev]: rews [B][Ntotal+1] (mean sample last); rng [B][2],
 * read and advanced in place to split(rng)[0]; Ybar and Ybar_out [B][Hn+1][nu]; noise_scale [Hn+1];
 * weights [B][Ntotal+1] out.  Uses the plan's partials and counters like the graph does, so it must
 * not run concurrently with dial_mpc_step on the same plan.  Fails for sharded plans
 * (Ntotal != Nsample) and for Ntotal + 1 > 131072. */
int dial_reverse_update_fused(dial_plan* plan, const float* rews, uint32_t* rng, const float* Ybar,
                              const float* noise_scale, float* Ybar_out, float* weights, void* stream);

/* qbar/qdbar/xbar (core/dial_core.py:133-135): weighted sums of this rank's stored
 * trajectories with `weights` [dev][Ntotal+1]; sharded runs sum the outputs across
 * ranks (the mean sample is counted on rank 0 only).  Outputs [dev]:
 * qbar [Hs+1,nq], qdbar [Hs+1,nv], xbar [Hs+1,nbody-1,3]. */
int dial_reverse_trajbar(dial_plan* plan, const float* weights, int rank,
                         float* qbar, float* qdbar, float* xbar, void* stream);

/* The stored trajectories of the LAST dial_reverse_rollout (the `pipeline_statess` that
 * core/dial_core.py:120-124 keeps alive: q, qd, x.pos of every sample): device-to-device copies
 * into caller buffers q [Nsample+1,Hs+1,nq], qd [..,nv], xpos [..,nbody-1,3] (each nullable). */
int dial_reverse_trajectories(dial_plan* plan, float* q, float* qd, float* xpos, void* stream);

/* ---- Multi-GPU reward exchange over NVLink peer memory (one process per GPU) -----------------
 * The reference is single-device; sharding the samples needs ONE exchange per reverse_once: all
 * ranks need all Ntotal rewards for std / softmax (core/dial_core.py:125-128).  Instead of a host-
 * issued collective the exchange is fused into the kernels on either side of it: the epilogue of
 * the rollout kernel stores each finished row's reward straight into the mailbox of EVERY rank
 * (peer stores through NVSwitch) and its last CTA raises a flag per rank; the weights kernel
 * spins on the W flags of its own mailbox (bounded), then reads the rewards locally.  The
 * info-only bars are summed the same way (push partial, flag, wait, add in rank order).  No host
 * round trip, no extra launch: a sharded control step is graph-capturable (dial_mpc_step).
 *   1. every rank: dial_exchange_create(plan, rank, world, handle)   -> 64-byte CUDA IPC handle
 *   2. all-gather the handles with any host transport (torch.distributed, MPI, a file)
 *   3. every rank: dial_exchange_connect(plan, handles[world][64])
 * From then on dial_reverse_rollout publishes, dial_reverse_update(_x) with rews_all == NULL
 * consumes, dial_reverse_trajbar returns the all-rank sums.  dial_exchange_status reads
 * {sequence, CTAs done, error (1 = a wait timed out after ~4 s), bars sequence, total ns the
 * update kernels waited for their slowest peer's flag, the same for the bars kernels}. */
int dial_exchange_create(dial_plan* plan, int rank, int world, unsigned char handle_out[DIAL_IPC_HANDLE_BYTES]);
int dial_exchange_connect(dial_plan* plan, const unsigned char* handles);
int dial_exchange_status(dial_plan* plan, uint32_t out[6]);

/* ---- Device-resident synchronous MPC loop -------------------------------------------------
 * The reference's main loop (core/dial_core.py:242-268) is, per control step,
 *     state = step_env(state, Y0[0]); Y0 = shift(Y0);
 *     for i < n_diffuse: rng, Y0, info = reverse_once(state, rng, Y0, noise[i])
 * with one jitted XLA program per piece.  Here the whole step is ONE CUDA graph: state, step
 * counters, rng and control knots stay in HBM (caller-owned `dial_mpc_buffers`), the key
 * splitting / shift / counter bookkeeping between kernels runs as tiny glue kernels, and
 * `dial_mpc_step` only replays the graph (captured on the second use of an
 * (n_diffuse, env_step) shape; the first use runs eagerly).  The graphs are captured again when the
 * launch sequence changes: a feature's first setting, or a change in the number of prediction launches or
 * in whether any instance predicts through its delay; other settings take effect at the next replay.
 * Results equal the eager
 * `dial_env_step` + `dial_reverse_*` sequence.  Sharded plans (Ntotal > Nsample) need a connected
 * exchange: every rank replays the same graph, the env step runs redundantly on every rank. */
typedef struct dial_mpc_buffers { /* all [dev], caller-owned, fixed while bound */
  float* qpos;            /* [nq]  state, advanced in place by the env step                  */
  float* qvel;            /* [nv]                                                            */
  float* qacc_warmstart;  /* [nv]                                                            */
  int32_t* counters;      /* [2]   info["step"], info["contact_stage"]; advanced in place    */
  uint32_t* rng;          /* [2]   planner rng; each reverse_once splits it                  */
  float* Y;               /* [Hn+1,nu] control knots, in/out                                 */
  float* ctrl;            /* [nu]  out: control applied by the env step                      */
  float* reward;          /* [1]   out: reward of the env step                               */
  float* rews;            /* [Nsample+1] out: this rank's sample rewards of the last reverse_once */
  float* rews_all;        /* [Ntotal+1]  out, sharded plans only (else NULL): all ranks' rewards  */
  float* qbar;            /* [Hs+1,nq]        nullable (all three or none): bars of the last  */
  float* qdbar;           /* [Hs+1,nv]        reverse_once                                    */
  float* xbar;            /* [Hs+1,nbody-1,3]                                                 */
  const float* noise;     /* [>= n_diffuse][Hn+1] annealing schedule (dial_core.py:259-261)  */
  /* Batched plans (n_inst = B > 1): every array above except noise gains a leading [B] dimension,
   * instance-major: qpos [B,nq], qvel/qacc_warmstart [B,nv], counters [B,2], rng [B,2],
   * Y [B,Hn+1,nu], ctrl [B,nu], reward [B], rews [B,Nsample+1], qbar [B,Hs+1,nq],
   * qdbar [B,Hs+1,nv], xbar [B,Hs+1,nbody-1,3].  rews_all must be NULL.  Instance b's results are
   * bitwise those of a single-instance plan bound to instance b's slices. */
  /* Per-instance tasks [B] (B = 1 for a single-instance plan), or NULL: every instance then plans the
   * task of the plan's own constants.  Non-NULL: every launch of dial_mpc_step (the env-step row and all
   * rollout rows) reads instance b's reward inputs from tasks[b], and the plan's task fields, including
   * what dial_plan_set_command / _set_stages put there, are ignored.  Instance b's results are bitwise
   * those of a plan whose constants hold tasks[b].  The captured graph holds the pointer, not the
   * contents: the caller may rewrite tasks between dial_mpc_step calls with a copy on the same stream
   * (stream-ordered, like dial_plan_set_command).  Each task must satisfy the ranges of dial_task. */
  const dial_task* tasks;
  /* Per-instance and ensemble models are not buffers: dial_plan_set_instance_model and
   * dial_plan_set_ensemble_model (below) write them into plan-owned arrays that dial_mpc_step reads.
   * With n_ens = K >= 1, rews [B,Nsample+1] receives each sample's score over its member rewards (the
   * member mean, or the measure dial_plan_set_ensemble_risk sets per instance), and
   * qbar / qdbar / xbar are the weighted means of member 0's trajectories: member 0 is the prediction
   * the caller reads. */
} dial_mpc_buffers;

/* Give instance b (0 <= b < n_inst; b = 0 for a single-instance plan) of the plan its own physical model
 * `m` [host], e.g. a payload on the base (body_mass, body_inertia, body_ipos), another floor friction
 * (pair_friction), joint damping, motor strength (actuator_gear) or gravity.  m must have the integer
 * structure of the plan's model (bodies, dofs, contact pairs, solver iteration counts, ...) and the same
 * timestep, jnt_range and actuator_ctrlrange (the plan descriptor holds copies of them); any other float
 * may differ.  Otherwise the call fails and dial_last_error names the first field that differs.  The
 * plan's gains, torque limits, joint ranges and dt stay shared by every instance.
 * Only dial_mpc_step reads per-instance models: the env-step row of instance b and, on a plan with
 * n_ens = 0, every rollout row of instance b; instance b's results are then bitwise those of a plan
 * created from m.  With n_ens >= 1 the instance model is the plant only (the env-step row); the rollout
 * rows run the member models of dial_plan_set_ensemble_model.  dial_env_step(_kin),
 * dial_pipeline_init, dial_rollout and the eager dial_reverse_* keep using the plan's own model.
 * The copy is stream-ordered on `stream`, out of plan-owned pinned staging, so it may be issued between
 * dial_mpc_step calls like dial_plan_set_command.  The first call on a plan allocates the per-instance
 * array (every slot starts as the plan's own model) and drops the captured graphs, which are captured
 * again on their next use; later calls do not.  Sharded plans (Ntotal != Nsample) reject the call.
 * Launches with per-instance models give each instance's rows CTAs of their own (each CTA stages one
 * model), with at most the warps per CTA of the default policy (dial_rollout_wpc). */
int dial_plan_set_instance_model(dial_plan* plan, int b, const dial_model_desc* m, void* stream);

/* Member k (0 <= k < n_ens) of instance b's planning ensemble on a plan with n_ens >= 1: the rollout
 * rows of member (b, k) run model `m` in every reverse_once of dial_mpc_step.  The same checks, errors
 * and stream-ordered copy out of plan-owned pinned staging as dial_plan_set_instance_model.  The first
 * call allocates the member array [n_inst * n_ens] (every slot starts as the plan's own model, not the
 * instance's) and drops the captured graphs; fails on a plan with n_ens == 0 and for b or k out of range.
 * n_ens = 1 with no member set plans on the plan's model, bitwise as n_ens = 0 without instance models:
 * the mismatch experiment, with the plant set by dial_plan_set_instance_model.  Launches with members
 * give each member's Nsample+1 rows CTAs of their own, as per-instance models do per instance. */
int dial_plan_set_ensemble_model(dial_plan* plan, int b, int k, const dial_model_desc* m, void* stream);

/* Risk measures of an ensemble plan: how instance b turns the K member rewards r_0..r_{K-1} of sample i
 * into its score rews[b][i] (dial_plan_set_ensemble_risk). */
#define DIAL_ENS_MEAN 0 /* (((r_0 + r_1) + ...) + r_{K-1}) / K in fp32, round-to-nearest: the default */
#define DIAL_ENS_CVAR 1 /* CVaR_alpha: the mean of the worst alpha-fraction of the members */

/* Instance b's risk measure on a plan with n_ens >= 1, from the next reverse_once of dial_mpc_step on.
 * mode DIAL_ENS_MEAN (alpha is ignored) or DIAL_ENS_CVAR with alpha finite and in (0, 1]; alpha <= 1/K
 * is the worst case, the minimum.  With t = alpha K in fp64, the host derives once:
 *   t <= 1 + 1e-6:                 n_tail = 1,        frac = 0,                 denom = 1
 *   |t - round(t)| <= 1e-6 K:      n_tail = round(t), frac = 0,                 denom = n_tail
 *   otherwise:                     n_tail = floor(t), frac = (float)(t - n_tail), denom = (float)t
 * and the reduction sorts the K rewards ascending (stable in member order: -0 stays before +0 if it
 * comes first), sets acc = s_0, adds s_1 .. s_{n_tail-1} in that order, adds fmul(frac, s_{n_tail})
 * when frac > 0 (a separate multiply and add), and writes acc / denom, all fp32 round-to-nearest.
 * CVaR with alpha = 1 is the mean up to rounding only (another summation order); DIAL_ENS_MEAN alone
 * reproduces a plan without the call.  A NaN member reward makes the score NaN; infinities go through
 * the arithmetic.  A non-finite score gets weight 0 in the update, as with the mean.
 * The copy of the 32-byte setting is stream-ordered on `stream`, out of plan-owned pinned staging that
 * dial_plan_create allocates with the setting array (n_ens >= 2; every instance starts at the mean), so
 * the call may be issued between dial_mpc_step calls.  The captured graphs read the array, so they are
 * kept: the setting takes effect at their next replay.  On a plan with n_ens = 1 any valid setting is
 * accepted and changes nothing (every measure of one reward is that reward).  Fails on a plan with
 * n_ens == 0, for b out of range, an unknown mode or a bad alpha. */
int dial_plan_set_ensemble_risk(dial_plan* plan, int b, int mode, float alpha, void* stream);

/* The member rewards of the last reverse_once of dial_mpc_step, out [dev] [n_inst, n_ens, Nsample+1]
 * (member k of instance b at (b n_ens + k)(Nsample+1)): the per-member rewards the risk measure reduced
 * (n_ens >= 2), or the bound rews (n_ens = 1).  A stream-ordered copy on `stream`.  Fails on a plan with
 * n_ens == 0 and before dial_mpc_bind. */
int dial_plan_member_rewards(dial_plan* plan, float* out, void* stream);

/* Adapting an ensemble plan (n_ens = K >= 2) to its plant.  Instance b keeps a belief over its K members:
 * log-weights L [K] in fp64 and w_k = (float) exp(L_k).  Every instance starts uniform.  While instance b
 * adapts, each dial_mpc_step with env_step == 1 first lets every member (b, k) make the plant's env step on
 * its own model, from the instance's pre-step state and counters with the action Y[b][0], and keeps its
 * post-step qvel vhat_k.  After the plant's step, with v its observed qvel, in fp64:
 *   e_k = sum_j ((vhat_kj - v_j) / sigma_j)^2  (j ascending, from the fp32 values)
 *   l_k = -min(e_k / 2, C), C = 1e4            (a NaN or infinite e_k gives -C: a NaN plant state
 *                                               shifts every member equally)
 *   L_k <- forget L_k + l_k;  L_k <- L_k - (M + log sum_k exp(L_k - M)), M = max_k L_k (member order).
 * With env_step 0 or 2, and on instances that do not adapt, the belief stays as it is.
 * An adapting instance scores each sample by its risk measure weighted by the belief.  Member k is kept
 * when w_k > 0 and w_k >= prune, or w_k is the largest weight; v_k = w_k for kept members, else 0, and
 * W = sum_k v_k in member order.  All fp32 round-to-nearest:
 *   DIAL_ENS_MEAN: (sum_k v_k r_k) / W, member order;
 *   CVaR, alpha K <= 1 + 1e-6 (the worst case): the minimum reward of the kept members;
 *   CVaR otherwise: tau = alpha W; over the (r, v) pairs sorted ascending by r (stable in member order),
 *     skipping v = 0, while m < tau: t = min(v_j, tau - m), acc += t r_j, m += t; the score is acc / m.
 * Sums start at -0.  A NaN reward of a kept member makes the score NaN; a pruned member's reward is never
 * read.  With uniform weights these equal the unweighted measures only up to rounding.  The GPU flushes
 * subnormal fp32 values to zero, so a weight below FLT_MIN counts as 0 there.
 * Each prediction is one more rollout launch over n_inst K rows and a small gather launch before the
 * plant's env step, and one belief launch after it: only in plans where some instance turned
 * adaptation on; a plan that never does keeps its launches. */

/* Instance b adapts (on = 1) or stops adapting (on = 0; the other arguments are then ignored and the
 * belief is kept).  forget in (0, 1], prune in [0, 1/K), sigma [host][nv] finite and > 0: the scale of
 * each qvel residual.  The 128-byte setting is copied stream-ordered on `stream` out of plan-owned pinned
 * staging, as for dial_plan_set_ensemble_risk.  The first call with on = 1 on a plan allocates the
 * prediction workspaces and drops the captured graphs; later calls keep them, and their setting takes
 * effect at the next replay.  Fails on a plan with n_ens < 2, for b out of range and for a bad argument,
 * which the error names. */
int dial_plan_set_ensemble_adapt(dial_plan* plan, int b, int on, float forget, float prune, const float* sigma,
                                 void* stream);

/* Instance b's belief from w [host][K]: each finite and >= 0, with a positive sum.  In fp64 the host
 * sets L_k = log(w_k / sum w) (-inf for w_k = 0: that member stays excluded) and w_k = (float) exp(L_k);
 * a stream-ordered copy on `stream`, as above.  The graphs are kept.  Lets an outside estimator drive the
 * belief where the plan does not step the plant (env_step 0). */
int dial_plan_set_ensemble_belief(dial_plan* plan, int b, const float* w, void* stream);

/* The current belief w [dev][n_inst, K] and the l [dev][n_inst, K] of each instance's last update (0
 * before the first), each nullable; stream-ordered copies on `stream`.  Fails on a plan with n_ens < 2. */
int dial_plan_ensemble_belief(dial_plan* plan, float* w, float* loglik, void* stream);

/* Per-instance sampling schedules of dial_mpc_step: instance b's softmax temperature, its noise rows and
 * how many diffusion iterations it runs.  In dial_mpc_step(plan, n, env_step), instance b runs the
 * iterations i < min(n, n_b) (n_b: its iteration limit, n when no limits are set), each with row i of its
 * own table and its own temperature when it has a schedule, else with the bound noise row i and the plan's
 * temp_sample.  In the iterations i >= min(n, n_b) instance b does nothing: none of its rollout rows run,
 * its rng is not split, and Y, rews, qbar / qdbar / xbar and the weights of the last iteration keep what its
 * last iteration produced (n_b = 0: it is only env-stepped and shifted).  Instance b then computes bitwise
 * what a single-instance plan with temp_sample = temp and the bound noise = its table computes with
 * dial_mpc_step(plan, min(n, n_b), env_step).  Every member of an ensemble instance uses the instance's
 * rows.  A plan on which neither call is ever made launches what it launched before.
 * Both calls copy stream-ordered on `stream` out of plan-owned pinned staging, so they may be issued
 * between dial_mpc_step calls.  The first call of each allocates its array and drops the captured graphs;
 * later calls keep them and take effect at the next replay.  Both reject sharded plans
 * (Ntotal != Nsample) and plans past the fused update (Ntotal + 1 > 131072).  dial_mpc_step fails, naming
 * the instance, when an instance with its own table would run more iterations than the table has rows,
 * and fails with DIAL_NO_FUSED_UPDATE set once either call has been made. */

/* Instance b's schedule: temp finite and > 0, noise [host][n_rows][Hn+1] finite with n_rows in 1..64.
 * noise == NULL returns instance b to the plan's temp_sample and the bound noise (temp and n_rows are then
 * ignored).  Fails for b out of range and for a bad argument, which the error names. */
int dial_plan_set_instance_schedule(dial_plan* plan, int b, float temp, int n_rows, const float* noise, void* stream);

/* The iteration limits n_iter [host][n_inst], each in 0..64.  While limits are set, the rollout launches
 * give each instance CTAs of its own (the layout of per-instance models, whose slots the first call
 * allocates with the plan's model when no model was set), so a skipped instance's CTAs exit whole; an
 * instance's results do not depend on the launch shape. */
int dial_plan_set_instance_iterations(dial_plan* plan, const int32_t* n_iter, void* stream);

/* Per-instance control latency of dial_mpc_step.  Instance b holds a FIFO queue of d_b actions [nu]
 * (d_b in 0..DIAL_MAXDELAY, 0 by default).  In a dial_mpc_step with env_step == 1 it pops the front a,
 * pushes Y[b][0] to the back (d_b = 0: a = Y[b][0]), and the plant's env step applies a: the action
 * planned at step t reaches the plant at step t + d_b.  ctrl and reward are those of that env step, and an
 * adapting ensemble instance scores its members' predictions under a too.  With env_step 0 or 2 the queue
 * does not move.
 * An instance that predicts (predict = 1, d_b >= 1) plans from a predicted state: in every dial_mpc_step,
 * after the env step and the shift, a copy of the plant's qpos, qvel, qacc_warmstart and counters takes d_b
 * env steps on the instance's planning model (its model; member (b, 0) of an ensemble plan) with the queued
 * actions in FIFO order, its task and counters advancing as the env step advances them.  Every rollout of
 * the instance starts from that state, so its rews, bars and knots describe the plan from it.  Without an
 * ensemble, the planning state recorded after step t equals, bit for bit, the plant state after step
 * t + d_b.  The other instances plan from the plant state.
 * The prediction is max d_b (over the predicting instances) rollout launches of one row per instance, each
 * skipping the instances whose prediction is shorter, after one copy of the plant state; a small queue
 * launch precedes the env step (and runs in steps without one while some instance predicts).  A plan on
 * which no delay is ever set launches what it launched before.  Sharded plans are rejected. */

/* Instance b's delay `steps` (0..DIAL_MAXDELAY) and `predict` (0 or 1).  Every call refills b's queue with
 * `steps` copies of Y[b][0] as it stands when the call's stream-ordered work runs on `stream` (so the plan
 * must be bound, dial_mpc_bind).  The first call allocates the queues and planning-state buffers.  The
 * graphs are captured again when the launch sequence changes: at the first call, and at a call that changes
 * the number of prediction launches or whether any instance predicts through its delay; other calls keep
 * them, and take effect at the next replay.  Fails for b out of range and for a bad argument, which the
 * error names. */
int dial_plan_set_instance_delay(dial_plan* plan, int b, int steps, int predict, void* stream);

/* Each instance's queue in application order: out [dev][n_inst][DIAL_MAXDELAY][nu], row j < d_b the action
 * the env step j + 1 steps from now applies, rows j >= d_b zero (all zero on a plan without delays).  A
 * stream-ordered copy on `stream`. */
int dial_plan_pending_actions(dial_plan* plan, float* out, void* stream);

/* The state the last planning rollouts of dial_mpc_step started from: qpos [dev][n_inst][nq], qvel and warm
 * [dev][n_inst][nv], counters [dev][n_inst][2] ({step, contact_stage}), each nullable; the predicted state of
 * a predicting instance, the plant state of every other.  Stream-ordered copies on `stream`. */
int dial_plan_planning_state(dial_plan* plan, float* qpos, float* qvel, float* warm, int32_t* counters, void* stream);

/* Per-instance observation of dial_mpc_step: instance b may plan from a noisy, late estimate of its plant
 * state instead of the state itself.  Its setting is an observation delay k_b in control steps, noise
 * standard deviations sigma_q[nv] (on qpos, in tangent space) and sigma_v[nv] (on qvel), and a noise key.
 * An instance observes while k_b > 0 or some sigma > 0; the plant, ctrl, reward and adaptation's belief
 * update keep the plant state.
 * History: each observing instance keeps a ring of plant records (qpos, qvel, qacc_warmstart, counters and
 * the action the env step applied: the front of its delay queue, else Y[b][0]).  A dial_mpc_step with
 * env_step == 1 pushes the post-step record.  A setting resets the ring; the next dial_mpc_step then seeds
 * it from the plant state.  With c_b records since the reset (the seed counted), the observed record is the
 * one age_b = min(k_b, c_b - 1) pushes back: the first k_b steps observe the oldest record there is.
 * Noise: each pushed or seeded record draws (key_b, sub) = split(key_b), eps = normal(sub, 2 nv) (JAX's
 * legacy Threefry sampler), and the observation is the observed record with hinge and slide qpos + sigma_q
 * eps[:nv], free-joint positions + sigma eps, a free (or ball) joint's quaternion
 * qnormalize(q * axisangle(w / |w|, |w|)) with w = sigma_rot eps in the body frame (physics_step's
 * composition), qvel + sigma_v eps[nv:], and the record's qacc_warmstart and counters.  A dof whose sigma
 * is 0 is copied bit for bit (a quaternion whose three sigma are 0 stays unnormalised); steps without an env
 * step reuse the last draw.
 * Planning: the instance's rollouts start from its observation.  One that predicts (its delay setting's
 * predict = 1) first takes age_b + d_b env steps on its planning model: the age_b actions applied since the
 * observed record, oldest first, then its d_b queued actions.  Without noise and without an ensemble its
 * planning state after step t equals the plant state after step t + d_b, bit for bit.
 * Launches: once some instance was given a setting, one observe launch runs after the env step and the
 * shift in every dial_mpc_step, in place of the copy of the plant state, followed by max(k_b + d_b) (over the
 * predicting instances) prediction launches of one row per instance.  A plan on which no observation is
 * ever set launches what it launched before.  k_b + d_b <= DIAL_MAXDELAY, checked by whichever of the two
 * setters runs second.  Sharded plans are rejected. */

/* Instance b's observation setting: `delay` (0..DIAL_MAXDELAY), qpos_std and qvel_std [host][nv] (each
 * nullable: zero), key [host][2] (nullable: {0, 0}).  A delay of 0 with every sigma 0 removes the setting:
 * the instance plans from its plant state again.  Every call resets b's ring and restarts its noise from
 * `key`, stream-ordered on `stream` (so the plan must be bound, dial_mpc_bind).  The first call allocates the
 * rings; it and a later call that changes the number of prediction launches make the graphs be captured
 * again; other calls keep them, and take effect at the next replay.  Fails for b out of range, a delay out of
 * range or one whose sum with b's action delay exceeds DIAL_MAXDELAY, a negative or non-finite sigma, and
 * sharded or unbound plans; the error names the bad argument. */
int dial_plan_set_instance_observation(dial_plan* plan, int b, int delay, const float* qpos_std,
                                       const float* qvel_std, const uint32_t key[2], void* stream);

/* The observation of the last dial_mpc_step, before the prediction: qpos [dev][n_inst][nq], qvel and warm
 * [dev][n_inst][nv], counters [dev][n_inst][2], age [dev][n_inst] (int32, the observed record's age), each
 * nullable; the plant state at age 0 for an instance that does not observe, and for every instance before
 * the first step after the first setting.  Stream-ordered copies on `stream`. */
int dial_plan_observed_state(dial_plan* plan, float* qpos, float* qvel, float* warm, int32_t* counters,
                             int32_t* age, void* stream);

/* One entry of an instance's push table (dial_plan_set_instance_pushes): after each env step of dial_mpc_step
 * whose post-step counter info["step"] lies in [step, step + n_steps), the plant takes the impulse of the
 * force `force` [N] applied at the point `pos` of body `body` and of the torque `torque` [N m], held for the
 * env step's duration.  pos is in the body's frame, force and torque in the world frame. */
typedef struct dial_push {
  int32_t step;      /* first post-step counter it fires at, >= 1 */
  int32_t n_steps;   /* env steps it fires in, >= 1 */
  int32_t body;      /* 1..nbody-1 (not the world) */
  float pos[3], force[3], torque[3];
} dial_push;

/* Per-instance pushes of dial_mpc_step: instance b's plant may be pushed between env steps, the standard test
 * of how well a controller recovers.  A push is an impulse on the plant state, applied after the env step
 * (and after adaptation's belief update) and before the shift, the observation and the prediction:
 *   qvel += M(q)^-1 J^T [torque; force] dt
 * with M the instance's plant mass matrix (armature included) at the post-step qpos, J the spatial Jacobian
 * (rotational rows, then translational) of the world point of `pos` on `body`, and dt = n_frames * timestep
 * the env step's duration; qpos is not changed.  Entries that fire in the same step add up.  A force held over
 * n env steps is a train of n impulses with the force's total impulse, each applied at the end of its step: the
 * physics steps inside an env step do not see it.  The reward of the env step at which a push fires does not
 * see it, the next one does; adaptation scores its members against the unpushed qvel; the observation ring and
 * the prediction start from the pushed state.  The planner is not told about pushes.  The trigger is the
 * plant's own counter, so a replayed graph needs no state of its own, and moving the counter (as a new bound
 * state does) moves the trigger with it.  Computed in fp64 from the fp32 state, then rounded once into qvel.
 * Launches: once some instance was given a table, one push launch runs after every env step; an instance with
 * no entry firing at its counter leaves it at entry.  A plan on which no table is ever set launches what it
 * launched before. */

/* Instance b's push table: n (0..DIAL_MAXPUSH) entries [host] (nullable when n = 0); n = 0 clears the table.
 * The copy is stream-ordered on `stream` (the plan must be bound, dial_mpc_bind).  The first table set on a plan
 * allocates the tables and drops the captured graphs; later calls keep them and take effect at the next
 * replay.  Fails for b out of range, n out of range, a body out of range or the world body, step < 1,
 * n_steps < 1, a non-finite pos, force or torque, and sharded or unbound plans; the error names the bad
 * argument. */
int dial_plan_set_instance_pushes(dial_plan* plan, int b, int n, const dial_push* pushes, void* stream);

/* One instance's plant fidelity (dial_plan_set_instance_plant): how finely its plant integrates and solves the
 * physics of an env step.  The planner's own settings are the plan model's timestep, iterations, ls_iterations
 * and tolerance with substeps 1. */
typedef struct dial_plant {
  int32_t substeps, iterations, ls_iterations;   /* 1..DIAL_MAXSUBSTEPS, 1..100, 1..50 */
  float tolerance;                                /* finite, >= 0 */
} dial_plant;

/* Per-instance plant fidelity of dial_mpc_step: instance b's plant may integrate the same physics more finely
 * and solve its contacts further than the planner's model, as a real robot or a finer simulator does.  With a
 * setting, instance b's env step makes substeps * n_frames physics steps of timestep / substeps on its plant
 * model: its instance model (dial_plan_set_instance_model) or the plan's model, with the setting's iterations,
 * ls_iterations and tolerance.  The control is computed once, from the pre-step state, and held across all of
 * them; the reward is computed once, on the post-step state; info["step"] and the env step's duration
 * n_frames * timestep (dial_plan_desc.dt) are unchanged.  Nothing else changes: the planner's rollouts,
 * ensemble members, adaptation's member steps, the prediction through a delay or observation and the push
 * impulse keep the plan's own discretisation.  substeps 1 with the plan model's solver settings computes
 * bitwise what an instance without a setting computes.
 * Launches: once some instance was given a setting, the plant's env step is one launch of the plan's generic
 * solver variant (never a shape-specialised kernel) per distinct substep count in use, each over every
 * instance with the others exiting at entry; an instance without a setting is in the group of substeps 1.  A
 * plan on which no setting is ever made launches what it launched before. */

/* Instance b's plant fidelity [host]; f = NULL clears it (b's plant then steps like its planner).  The copies
 * are stream-ordered on `stream` (the plan must be bound, dial_mpc_bind).  The first setting on a plan
 * allocates the plant model slots and drops the captured graphs, and so does any later call that changes the
 * set of distinct substep counts in use; other calls keep them and take effect at the next replay.  A later
 * dial_plan_set_instance_model(b) reaches b's plant with its fidelity kept.  Fails for b out of range, a field
 * out of range, and sharded or unbound plans; the error names the bad argument. */
int dial_plan_set_instance_plant(dial_plan* plan, int b, const dial_plant* f, void* stream);

/* One instance's terrain (dial_plan_set_instance_terrain): a grid of nx x ny heights h[j][i] (row-major, j the
 * y index), 2..DIAL_MAXTERRAIN per side, spacing > 0, origin (x0, y0).  Vertex (i, j) is the world point
 * (x0 + i spacing, y0 + j spacing, h[j][i]); heights are absolute world z. */
typedef struct dial_terrain {
  int32_t nx, ny;
  float x0, y0, spacing;
  const float* heights;   /* [ny][nx], host memory */
} dial_terrain;

/* Per-instance terrain of dial_mpc_step.  For an instance with a terrain on a side, the terrain replaces every
 * plane geom on the world body in that side's env steps.  Each cell is split along the diagonal from (i, j) to
 * (i+1, j+1) into two triangles; H(x, y) is the piecewise linear surface.  A sphere (centre c, radius r) of a
 * floor pair, and each end sphere of a capsule on one, is tested against the plane of the triangle under
 * (c.x, c.y): with that triangle's slopes (sx, sy), n = (-sx, -sy, 1) / |.| (exactly (0, 0, 1) when both are
 * 0), dist = dot(c - (c.x, c.y, H(c.x, c.y)), n) - r, and the contact point and frame follow the plane's
 * formulas with that n.  Outside the grid the query point is clamped into it and the plane is horizontal at H
 * of the clamped point.  Every floor pair keeps its contact slots, so the contact counts and the solver are
 * those of the flat floor.  The model is locally planar: it holds where the surface varies slowly at the scale
 * of a foot, not at steps (a sphere only sees the triangle beneath its centre).  The built-in rewards measure
 * their base height (Go2 walk, H1 walk, H1 loco) and Go2 walk's foot heights above H beneath; custom rewards
 * read it with dial_terrain_height (include/dial_custom_reward.h).
 * Side DIAL_TERRAIN_PLANT is read by the plant's env step (every plant-fidelity launch), side
 * DIAL_TERRAIN_PLANNER by the planner's rollouts, the ensemble members, adaptation's member steps and the
 * prediction launches.  Launches that read a terrain run the terrain build of the plan's solver variant (the
 * generic star<3,6> kernel on a Go2 plan); rows without a terrain compute there bitwise what they compute in
 * the plan's other kernels.  A plan on which no terrain is ever set launches what it launched before. */

/* Instance b's terrain on `side` [host]; t = NULL makes that side flat.  The heights are copied into
 * plan-owned device memory, stream-ordered on `stream` (the plan must be bound, dial_mpc_bind).  The first
 * terrain on a side drops the captured graphs, and so does a table larger than b's allocation on that side;
 * other calls keep them and take effect at the next replay.  Fails for b or side out of range, a grid size out
 * of range, a spacing that is not finite and > 0, a height that is not finite, a model without a floor pair
 * (a plane geom on the world body), the dense solver path, and sharded or unbound plans; the error names the
 * bad argument. */
int dial_plan_set_instance_terrain(dial_plan* plan, int b, int side, const dial_terrain* t, void* stream);

/* Bind the state block; M_shift [host][Hn+1][Hn+1] = u2node . roll(-1, last row 0) . node2u
 * (MBDPI.shift, core/dial_core.py:160-165), shared by all instances of a batched plan.  Drops
 * previously captured graphs. */
int dial_mpc_bind(dial_plan* plan, const dial_mpc_buffers* buffers, const float* M_shift);

/* One control step on `stream`: [env_step == 1: state <- env.step(state, Y[0])], [env_step == 1
 * or 2: Y <- shift(Y)], then n_diffuse x reverse_once with noise rows 0..n_diffuse-1.
 * env_step = 0 plans from the bound state as it is (deploy/dial_plan.py: the state comes from
 * the robot); env_step = 2 shifts and plans without advancing the state (a planner whose state
 * is written by somebody else once per control period). */
int dial_mpc_step(dial_plan* plan, int n_diffuse, int env_step, void* stream);
/* A batched plan advances all B loops in the same graph: the env step rolls B rows, the shift runs
 * one CTA per instance, every reverse_once is one rollout launch over B (Nsample+1) rows and one
 * fused update launch over B instances.  With n_ens = K >= 2 the rollout covers B K (Nsample+1) rows,
 * row ((b K) + k)(Nsample+1) + i, and one more small launch reduces the members' rewards into rews
 * under each instance's risk measure.  DIAL_NO_FUSED_UPDATE is an error on a batched plan.  The
 * eager dial_reverse_rollout / _update(_x) / _trajbar / _trajectories reject batched plans;
 * dial_rollout, dial_env_step(_kin) and dial_pipeline_init keep their single-instance meaning. */

/* jax.random.split(rng) / the planner's key threading (core/dial_core.py:106,145):
 * host-side Threefry-2x32; out[0] is the new rng, out[1] the sampling key. */
void dial_key_split(const uint32_t key[2], uint32_t out0[2], uint32_t out1[2]);

/* tuning aid: with DIAL_DEBUG_COUNTERS=1 in the environment at plan creation the dense solver
 * path counts [0] physics steps and [1] Newton iterations; reads and resets the counters. */
int dial_debug_counters(dial_plan* plan, float out[8]);

/* Which solver instantiation `model` maps to (1 star<3,6>, 2 star<5,7>, 3 dense nv=22,
 * 4 star<5,6>, 0 generic tree, <0 unsupported): custom-reward builds compile only this one
 * (-DDIAL_ONLY_VARIANT=v). */
int dial_solver_variant(const dial_model_desc* model);

/* The rollout kernel `plan` launches: "v<variant>" (the generic instantiation of its solver variant,
 * see dial_solver_variant) or the name of a kernel specialised on the integer structure of one model
 * ("go2": the stock Go2 scene), chosen at plan creation when every value it fixes equals the plan's
 * own; DIAL_FORCE_GENERIC_SHAPE=1 at plan creation keeps the generic one.
 * "" for a null plan. */
const char* dial_plan_rollout_kernel(const dial_plan* plan);

/* "" for the stock library; the identifier (-DDIAL_CUSTOM_REWARD_ID) of the reward source a
 * custom build was compiled with.  Only such a build accepts env_id == DIAL_ENV_CUSTOM. */
const char* dial_custom_reward_id(void);

/* Measured fp32 FFMA throughput of the current device in TFLOP/s (independent FMA chains at full
 * occupancy, best of 3, CUDA events; synchronous): the roofline denominator bench.py reports the
 * rollout kernel's flop rate against.  iters = loop trips of 128 FFMAs per thread. */
int dial_fp32_peak(int iters, float* tflops_out);

/* kernel launches issued by this plan since creation (bench bookkeeping) */
int64_t dial_launch_count(const dial_plan* plan);
/* Warps per CTA of the default rollout launch policy for `nrows` rows (grid = ceil(nrows / wpc));
   DIAL_WPC overrides it at launch.  0 for a null plan or nrows < 1. */
int dial_rollout_wpc(const dial_plan* plan, int nrows);

#ifdef __cplusplus
}
#endif
#endif /* DIAL_B200_H_ */
