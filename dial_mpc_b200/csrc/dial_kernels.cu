// dial_kernels.cu — sm_90a kernels + the C ABI of include/dial_b200.h.
//
// Kernels
//   rollout_kernel<WPC>   one warp per sample row, persistent over the horizon; the
//                         compiled model + plan constants are staged into shared memory
//                         with one TMA bulk copy (cp.async.bulk + mbarrier) per CTA.
//   weights_kernel        population std + max-subtracted softmax over all rewards
//                         (warp-shuffle + one smem stage reductions), single CTA.
//   ybar_kernel           Ybar = sum_n w_n Y0s_n with Y0s regenerated from eps / Threefry;
//                         per-CTA partials, last CTA reduces in fixed order (deterministic).
//   trajbar_kernel        qbar / qdbar / xbar weighted sums over the stored trajectories.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <float.h>
#include <cmath>
#include <memory>
#include <string>
#include <vector>
#include <new>
#include "dial_host.h"
#define DIAL_STR2(x) #x
#define DIAL_STR(x) DIAL_STR2(x)

static thread_local std::string g_err;
static int fail(const std::string& s) { g_err = s; return -1; }
#define CUDA_OK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(std::string(#x) + ": " + cudaGetErrorString(e_)); } while (0)

// The rollout kernel lives in dial_rollout_variant.cu, compiled once per solver variant
// (-DDIAL_VARIANT=v) so that the five instantiations build in parallel; each object exports
// one launcher.  Custom-reward builds (-DDIAL_ONLY_VARIANT=v) compile a single translation unit, whose one
// launcher (DIAL_V_LAUNCHER) is the terrain build when compiled with DIAL_TERRAIN.
typedef cudaError_t (*dial_launch_fn)(const DevModel*, const DevPlan*, const RolloutArgs&, int, int, size_t, cudaStream_t);
#ifdef DIAL_ONLY_VARIANT
#define DIAL_VARIANT DIAL_ONLY_VARIANT
#include "dial_rollout_variant.cu"
#else
#define DIAL_DECL_LAUNCH(s) cudaError_t dial_launch_rollout_##s(const DevModel*, const DevPlan*, const RolloutArgs&, int, int, size_t, cudaStream_t);
DIAL_DECL_LAUNCH(v0) DIAL_DECL_LAUNCH(v1) DIAL_DECL_LAUNCH(v2) DIAL_DECL_LAUNCH(v3) DIAL_DECL_LAUNCH(v4)
// Terrain builds (dial_rollout_variant.cu with -DDIAL_TERRAIN) of every variant but the dense one, which has
// none: the launches that read a terrain (dial_plan_set_instance_terrain) run them.
DIAL_DECL_LAUNCH(v0_terrain) DIAL_DECL_LAUNCH(v1_terrain) DIAL_DECL_LAUNCH(v2_terrain) DIAL_DECL_LAUNCH(v4_terrain)
// Shape-specialised star<3,6> kernels (dial_rollout_variant.cu with -DDIAL_SHAPE_NAME=s): the stock Go2
// scene, with the structure values that dial_mpc_b200.modelc.shape derives from its model.  A plan launches one only when dial_shape_matches_<s> finds every fixed
// value equal to its own model and plan.  Custom-reward builds hold none.
#define DIAL_DECL_SHAPE(s) DIAL_DECL_LAUNCH(s) bool dial_shape_matches_##s(const DevModel&, const dial_plan_desc&);
DIAL_DECL_SHAPE(go2)
static const struct {
  const char* name;
  dial_launch_fn launch;
  bool (*matches)(const DevModel&, const dial_plan_desc&);
} kShapes[] = {{"go2", dial_launch_rollout_go2, dial_shape_matches_go2}};
#endif

// ---------------------------------------------------------------------------------
// softmax weights over all rewards (core/dial_core.py:125-128), single CTA
// ---------------------------------------------------------------------------------
// block-wide sum of K values per thread (+ optionally the max of one): shuffle tree, one smem
// stage, result identical in every thread.  T = double: 64-bit shuffles (the reward statistics).
template <typename T, int K>
__device__ __forceinline__ void block_reduce(T (&v)[K], T* mx, T* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (mx) *mx = fmax(*mx, __shfl_xor_sync(0xffffffffu, *mx, o));
  }
  __syncthreads();   // previous use of `red` is over
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) red[k * 32 + wid] = v[k];
    if (mx) red[K * 32 + wid] = *mx;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = lane < nw ? red[k * 32 + lane] : T(0);
  if (mx) *mx = lane < nw ? red[K * 32 + lane] : T(-INFINITY);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (mx) *mx = fmax(*mx, __shfl_xor_sync(0xffffffffu, *mx, o));
  }
}

// rews [n] (mean sample last) -> weights [n] = softmax((rews - rews[n-1]) / std(rews) / temp)
// (core/dial_core.py:125-128).  Deviations from the reference, which has no guards (SURVEY Appendix F):
//   * non-finite rewards (diverged samples) get weight 0 and are left out of the statistics;
//   * std == 0 (all finite rewards equal, e.g. zero noise): uniform weights over the finite
//     samples instead of 0/0 = NaN;
//   * no finite reward at all: the whole weight goes to the mean sample (Ybar is kept);
//   * a non-finite rbar only changes the reference point of the shift (softmax is shift-invariant).
// One function computes the statistics for both kernels that use them (weights_kernel and the fused
// update_kernel), so the eager update and the control-step graph cannot drift apart.  The kernels
// compute the logit of sample i as (r_i - shift) * inv - mx.
struct SoftmaxParams {
  float shift, inv, mx;   // inv = 1 / std / temp, 0 when the finite rewards are flat (uniform weights)
  bool none;              // no finite reward
};
// Pass 2 of reward_softmax_params (ill-conditioned rewards): the deviations from the pass-1 mean
// (rbar + mean), summed and block-reduced in fp64.  Not inlined: the fp64 registers of this rare path
// stay out of the register allocation of the kernels' common path.
__device__ __noinline__ SoftmaxParams reward_softmax_params_fp64(const float* __restrict__ rews, int n, float temp,
                                                                 float rbar, float mean, float cnt, float* red_f) {
  double* red = reinterpret_cast<double*>(red_f);
  SoftmaxParams s;
  s.none = false;
  const double c = isfinite(mean) ? (double)rbar + (double)mean : 0.0;
  double s1[1] = {0.0}, s2[1] = {0.0}, rmax = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float r = __ldcg(rews + i);
    if (isfinite(r)) { const double d = (double)r - c; s1[0] += d; s2[0] += d * d; rmax = fmax(rmax, (double)r); }
  }
  block_reduce<double, 1>(s1, &rmax, red);      // two reductions: `red` holds 2 x 32 doubles
  block_reduce<double, 1>(s2, nullptr, red);
  const double m = s1[0] / (double)cnt, var64 = s2[0] / (double)cnt - m * m;
  s.shift = (float)rmax;   // the logit of the largest reward is 0; (r - rmax) is exact near the top
  s.mx = 0.f;
  // (clamped: a std of a few denormal ulp would give inf, and 0 * inf = NaN for the max sample)
  s.inv = var64 > 0.0 ? (float)fmin(1.0 / (sqrt(var64) * (double)temp), 3.4028234663852886e38) : 0.f;
  return s;
}
// Pass 1: count, sum and sum of squares of d = r - rbar and the max of d over the finite rewards, in
// fp32 (rbar = 0 when it is not finite).  The one-pass variance is accurate while the shift lies near
// the bulk of the rewards: it is used when rbar is finite, nothing overflowed and the shift is within
// 8 standard deviations of the mean (|mean(d)| <= 8 std), where it loses at most 6 bits.  Otherwise it
// cancels: with a NaN mean row, rewards -8 +- 0.003 gave a std of exactly 0, -30 +- 0.01 one 21 % off;
// a mean sample 1e4 spreads below the others put it 1 % off at 2^17 rewards; a finite reward beyond
// 1.8e19 overflowed d^2 (std = inf, every sample the same weight).  Those rewards take pass 2: the
// deviations from the pass-1 mean, summed and block-reduced in fp64 (no cancellation, no overflow for
// fp32 rewards), and logits relative to the largest finite reward.  The branch is uniform across the
// block (every thread holds the same sums).  `red`: shared memory for 4 x 32 floats.
__device__ __forceinline__ SoftmaxParams reward_softmax_params(const float* __restrict__ rews, int n, float temp,
                                                               float* red) {
  float rbar = __ldcg(rews + n - 1);
  const bool rbar_finite = isfinite(rbar);
  if (!rbar_finite) rbar = 0.f;
  float st[3] = {0.f, 0.f, 0.f}, dmax = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float r = __ldcg(rews + i);
    if (isfinite(r)) { const float d = r - rbar; st[0] += 1.f; st[1] += d; st[2] += d * d; dmax = fmaxf(dmax, d); }
  }
  block_reduce<float, 3>(st, &dmax, red);
  SoftmaxParams s;
  const float cnt = st[0];
  s.none = cnt == 0.f;
  const float mean = st[1] / fmaxf(cnt, 1.f);
  const float var = st[2] / fmaxf(cnt, 1.f) - mean * mean;
  const float sd = sqrtf(fmaxf(var, 0.f));
  if (s.none || (rbar_finite && isfinite(st[2]) && fabsf(mean) <= 8.f * sd)) {
    s.shift = rbar;
    s.inv = (sd > 0.f) ? 1.f / sd / temp : 0.f;
    s.mx = dmax * s.inv;
    return s;
  }
  return reward_softmax_params_fp64(rews, n, temp, rbar, mean, cnt, red);
}

// Multi-GPU consumer side of the reward exchange (dial_exchange_*): wait until every rank's flag
// in the local mailbox carries the current sequence number.  Bounded spin (~4 s of %globaltimer):
// a peer that never arrives sets *err instead of hanging the GPU.
struct XchWait {
  const float* mbox;            // local mailbox [2][n]; null: no exchange, `rews` is used as given
  const uint32_t* flags;        // local flags [2][DIAL_MAXRANK]
  uint32_t* seq;                // local sequence number, bumped when the weights are done
  uint32_t* err;                // local error word (1: timeout)
  float* rews_copy;             // optional compact copy of the gathered rewards [n]
  int world;
};
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// `acc` (nullable): running total of the time this rank spent waiting for its slowest peer, in ns
// (dial_exchange_status words 4 / 5) — the part of a sharded step that is skew + NVLink latency.
__device__ __forceinline__ void xch_wait_flags(const uint32_t* flags, uint32_t want, int world, uint32_t* err,
                                               uint32_t* acc = nullptr) {
  if ((int)threadIdx.x < world) {
    const volatile uint32_t* f = flags + threadIdx.x;
    const unsigned long long t0 = globaltimer_ns();
    while (*f < want) {
      if (globaltimer_ns() - t0 > 4000000000ull) { *err = 1u; break; }
      __nanosleep(100);
    }
    if (acc) {
      const unsigned long long dt = globaltimer_ns() - t0;
      const unsigned m = __reduce_max_sync(__activemask(), (unsigned)(dt > 0xffffffffull ? 0xffffffffull : dt));
      if (threadIdx.x == 0) *acc += m;
    }
    __threadfence_system();
  }
  __syncthreads();
}

__global__ void __launch_bounds__(1024) weights_kernel(const float* __restrict__ rews, int n, float temp,
                                                        float* __restrict__ weights, const XchWait X) {
  __shared__ __align__(8) float red[4 * 32];
  const int tid = threadIdx.x;
  if (X.mbox) {
    const uint32_t seq = *X.seq, buf = seq & 1u;
    xch_wait_flags(X.flags + buf * DIAL_MAXRANK, seq + 1u, X.world, X.err, X.err + 2);
    rews = X.mbox + (size_t)buf * n;
    if (X.rews_copy)
      for (int i = tid; i < n; i += blockDim.x) X.rews_copy[i] = __ldcg(rews + i);
  }
  const SoftmaxParams s = reward_softmax_params(rews, n, temp, red);
  if (s.none) {
    for (int i = tid; i < n; i += blockDim.x) weights[i] = (i == n - 1) ? 1.f : 0.f;
    if (X.mbox && tid == 0) *X.seq = *X.seq + 1u;
    return;
  }
  float z[1] = {0.f};
  for (int i = tid; i < n; i += blockDim.x) {
    const float r = __ldcg(rews + i);
    const float e = isfinite(r) ? expf((r - s.shift) * s.inv - s.mx) : 0.f;   // flat: inv = 0, every logit 0
    weights[i] = e;
    z[0] += e;
  }
  block_reduce<float, 1>(z, nullptr, red);
  const float iz = 1.f / z[0];
  for (int i = tid; i < n; i += blockDim.x) weights[i] *= iz;
  if (X.mbox && tid == 0) *X.seq = *X.seq + 1u;   // the next reverse_once uses the other mailbox half
}

// Sum of the per-rank partial bars (qbar|qdbar|xbar, core/dial_core.py:133-135) over NVLink peer
// memory: push my partial into slot [rank] of every rank's bars mailbox, raise my flag there,
// wait for all flags here, add the slots in rank order (bitwise identical on every rank).
struct BarsXch {
  float* mbox[DIAL_MAXRANK];        // bars mailbox of rank p: [2][DIAL_MAXRANK][nbar]
  uint32_t* flags[DIAL_MAXRANK];    // bars flags of rank p:   [2][DIAL_MAXRANK]
  uint32_t* seq;                    // local bars sequence number
  uint32_t* err;
  int world, rank, nbar;
  const float* partial;             // local partial [nbar]
  float* out[3];
  int n0, n1;                       // nbar = n0 (q) + n1 (qd) + rest (x)
};
__global__ void __launch_bounds__(1024) bars_allreduce_kernel(const BarsXch B) {
  const uint32_t seq = *B.seq, buf = seq & 1u;
  const size_t half = (size_t)buf * DIAL_MAXRANK * B.nbar;
  for (int p = 0; p < B.world; ++p) {
    float* dst = B.mbox[p] + half + (size_t)B.rank * B.nbar;
    for (int i = threadIdx.x; i < B.nbar; i += blockDim.x) dst[i] = B.partial[i];
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    for (int p = 0; p < B.world; ++p)
      *reinterpret_cast<volatile uint32_t*>(B.flags[p] + buf * DIAL_MAXRANK + B.rank) = seq + 1u;
  }
  __syncthreads();
  xch_wait_flags(B.flags[B.rank] + buf * DIAL_MAXRANK, seq + 1u, B.world, B.err, B.err + 3);
  const float* mine = B.mbox[B.rank] + half;
  for (int i = threadIdx.x; i < B.nbar; i += blockDim.x) {
    float s_ = 0.f;
    for (int p = 0; p < B.world; ++p) s_ += __ldcg(mine + (size_t)p * B.nbar + i);
    float* o = i < B.n0 ? B.out[0] + i : (i < B.n0 + B.n1 ? B.out[1] + (i - B.n0) : B.out[2] + (i - B.n0 - B.n1));
    *o = s_;
  }
  __syncthreads();
  if (threadIdx.x == 0) *B.seq = seq + 1u;
}

// sum_b col[b * stride], b = 0..count-1, in that order, with 16 independent L2 loads in flight (the
// last-CTA reductions of ybar_kernel / update_kernel: a plain loop pays one L2 round trip per term)
__device__ __forceinline__ float ordered_column_sum(const float* __restrict__ col, int stride, unsigned count, bool on) {
  float tot = 0.f;
  if (!on) return tot;
  unsigned b = 0;
  for (; b + 16 <= count; b += 16) {
    float v[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) v[k] = __ldcg(col + (size_t)(b + k) * stride);
#pragma unroll
    for (int k = 0; k < 16; ++k) tot += v[k];
  }
  for (; b < count; ++b) tot += __ldcg(col + (size_t)b * stride);
  return tot;
}

// ---------------------------------------------------------------------------------
// Ybar = sum_n w_n * Y0s_n  (core/dial_core.py:129-132), Y0s regenerated
// ---------------------------------------------------------------------------------
#define YBAR_THREADS 256
__global__ void __launch_bounds__(YBAR_THREADS) ybar_kernel(const float* __restrict__ weights, const float* __restrict__ eps,
                                                             uint32_t key0, uint32_t key1, const float* __restrict__ Ybar,
                                                             const float* __restrict__ noise, int Ntotal, int Hn1, int nu,
                                                             float* __restrict__ partial, unsigned int* __restrict__ counter,
                                                             float* __restrict__ Ybar_out,
                                                             const uint32_t* __restrict__ key_dev) {
  if (key_dev) { key0 = key_dev[0]; key1 = key_dev[1]; }
  // thread -> (sample slot, output element); elements = Hn1*nu <= 160
  const int ne = Hn1 * nu;
  __shared__ float acc[YBAR_THREADS];
  __shared__ bool is_last;
  const int slots = YBAR_THREADS / ne;  // samples processed concurrently per CTA
  const int slot = threadIdx.x / ne, el = threadIdx.x - slot * ne;
  float a = 0.f;
  if (slot < slots) {
    const int k = el / nu;
    const float yb = Ybar[el], ns = noise[k];
    const uint32_t ntot = (uint32_t)Ntotal * (uint32_t)ne;
    for (int n = blockIdx.x * slots + slot; n <= Ntotal; n += gridDim.x * slots) {
      float y = yb;
      if (n < Ntotal && k > 0) {
        uint32_t idx = (uint32_t)n * (uint32_t)ne + (uint32_t)el;
        float e = eps ? eps[idx] : jax_normal_legacy(key0, key1, idx, ntot);
        y = e * ns + yb;
      }
      y = fminf(fmaxf(y, -1.f), 1.f);
      a += weights[n] * y;
    }
  }
  acc[threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.x < ne) {
    float s = 0.f;
    for (int sl = 0; sl < slots; ++sl) s += acc[sl * ne + threadIdx.x];
    partial[blockIdx.x * ne + threadIdx.x] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (is_last) {
    if (threadIdx.x < ne) Ybar_out[threadIdx.x] = ordered_column_sum(partial + threadIdx.x, ne, gridDim.x, true);
    if (threadIdx.x == 0) *counter = 0u;
  }
}

// ---------------------------------------------------------------------------------
// Fused update of the control step graph: weights + Ybar + rng advance in ONE multi-CTA kernel
// (dial_core.py:106,125-132).  Every CTA recomputes the reward statistics (n <= 131072: up to 512
// L2-resident loads per thread at the 65536-sample config, a few at 2048), accumulates sum_n e_n Y0s_n and sum_n e_n over its share of the samples with
// e_n = exp((r_n - rbar) / std / temp - max) (reward_softmax_params); the last CTA adds the partials in fixed order,
// divides, normalises the stored weights, and advances the planner rng.  Two graph nodes fewer per
// reverse_once (a launch boundary inside a graph costs about a microsecond, so this is about graph
// size and the host-visible weights dependency more than time).
// Batched plans: blockIdx.y is the instance; each instance runs the single-instance grid on its own
// slices of rews / weights / rng / Ybar / partials / counter, so its arithmetic and order are unchanged.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(YBAR_THREADS) update_kernel(const float* __restrict__ rews, int n, float temp,
                                                               float* __restrict__ weights, const XchWait X,
                                                               uint32_t* __restrict__ rng, const float* __restrict__ Ybar,
                                                               const float* __restrict__ noise, int Ntotal, int Hn1, int nu,
                                                               float* __restrict__ partial, unsigned int* __restrict__ counter,
                                                               float* __restrict__ Ybar_out, const InstSchedule* __restrict__ sched,
                                                               const int32_t* __restrict__ iter_lim, int iter,
                                                               const float* weights_prev) {
  __shared__ __align__(8) float red[4 * 32];
  __shared__ float acc[YBAR_THREADS];
  __shared__ bool is_last;
  const int tid = threadIdx.x;
  {
    const size_t b = blockIdx.y, ne1 = (size_t)Hn1 * nu;
    rews += b * n; weights += b * n; rng += 2 * b; Ybar += b * ne1; Ybar_out += b * ne1;
    partial += b * gridDim.x * (ne1 + 1); counter += b;
    if (!schedule_runs(iter_lim, b, iter)) {
      // instance b is past its iteration limit: its knots and its last iteration's weights move on to this
      // iteration's buffers unchanged; rng and counter stay as they are
      if (blockIdx.x == 0)
        for (int i = tid; i < (int)ne1; i += blockDim.x) Ybar_out[i] = Ybar[i];
      if (weights_prev != weights - b * n)
        for (int i = blockIdx.x * blockDim.x + tid; i < n; i += gridDim.x * blockDim.x) weights[i] = weights_prev[b * n + i];
      return;
    }
    if (sched && sched[b].on) { temp = sched[b].temp; noise = sched[b].noise[iter]; }
  }
  if (X.mbox) {
    const uint32_t seq = *X.seq, buf = seq & 1u;
    xch_wait_flags(X.flags + buf * DIAL_MAXRANK, seq + 1u, X.world, X.err, blockIdx.x == 0 ? X.err + 2 : nullptr);
    rews = X.mbox + (size_t)buf * n;
  }
  uint32_t key0, key1;
  const uint32_t r0 = rng[0], r1 = rng[1];
  split_key(r0, r1, key0, key1);
  // ---- softmax parameters over the finite rewards (the same function as weights_kernel) -----------
  const SoftmaxParams sp = reward_softmax_params(rews, n, temp, red);
  // ---- this CTA's share of sum e_n Y0s_n (thread -> (sample slot, knot element)) and sum e_n ------------
  const int ne = Hn1 * nu;
  const int slots = YBAR_THREADS / ne;
  const int slot = tid / ne, el = tid - slot * ne;
  float a = 0.f, z = 0.f;
  if (slot < slots) {
    const int k = el / nu;
    const float yb = Ybar[el], ns = noise[k];
    const uint32_t ntot = (uint32_t)Ntotal * (uint32_t)ne;
    for (int s_ = blockIdx.x * slots + slot; s_ <= Ntotal; s_ += gridDim.x * slots) {
      const float r = __ldcg(rews + s_);
      float e = isfinite(r) ? expf((r - sp.shift) * sp.inv - sp.mx) : 0.f;
      if (sp.none) e = (s_ == Ntotal) ? 1.f : 0.f;          // no finite reward: keep the mean sample
      float y = yb;
      if (s_ < Ntotal && k > 0) {
        const uint32_t idx = (uint32_t)s_ * (uint32_t)ne + (uint32_t)el;
        y = jax_normal_legacy(key0, key1, idx, ntot) * ns + yb;
      }
      y = fminf(fmaxf(y, -1.f), 1.f);
      a += e * y;
      if (el == 0) { z += e; weights[s_] = e; }
    }
  }
  acc[tid] = a;
  float zz[1] = {z};
  block_reduce<float, 1>(zz, nullptr, red);
  __syncthreads();
  if (tid < ne) {
    float s_ = 0.f;
    for (int sl = 0; sl < slots; ++sl) s_ += acc[sl * ne + tid];
    partial[blockIdx.x * (ne + 1) + tid] = s_;
  }
  if (tid == 0) partial[blockIdx.x * (ne + 1) + ne] = zz[0];
  __threadfence();
  __syncthreads();
  if (tid == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // one thread per column of the partials (columns 0..ne-1: sum e Y0s, column ne: sum e), one pass,
  // 16 L2 loads in flight, added in CTA order (bitwise deterministic)
  __shared__ float zsh;
  float tot = ordered_column_sum(partial + tid, ne + 1, gridDim.x, tid <= ne);
  if (tid == ne) zsh = tot;
  if (ne == (int)blockDim.x && tid == 0) zsh = ordered_column_sum(partial + ne, ne + 1, gridDim.x, true);
  __syncthreads();
  const float iz = 1.f / zsh;
  if (tid < ne) Ybar_out[tid] = tot * iz;
  for (int i = tid; i < n; i += blockDim.x) {
    weights[i] = __ldcg(weights + i) * iz;
    if (X.mbox && X.rews_copy) X.rews_copy[i] = __ldcg(rews + i);
  }
  if (tid == 0) {
    *counter = 0u;
    uint32_t n0, n1;
    split_rng(r0, r1, n0, n1);
    rng[0] = n0; rng[1] = n1;
    if (X.mbox) *X.seq = *X.seq + 1u;
  }
}

// ---------------------------------------------------------------------------------
// glue of the device-resident MPC loop (dial_mpc_step): everything the reference's Python loop
// does between kernels (core/dial_core.py:242-268) as tiny kernels, so that one MPC step is one
// CUDA graph with no host work inside
// ---------------------------------------------------------------------------------
// rng, key = jax.random.split(rng)   (dial_core.py:106), legacy layout as dial_key_split
__global__ void mpc_split_kernel(uint32_t* __restrict__ rng, uint32_t* __restrict__ key) {
  if (threadIdx.x == 0) {
    const uint32_t k0 = rng[0], k1 = rng[1];
    uint32_t a0 = 0, b0 = 2, a1 = 1, b1 = 3;
    threefry2x32(k0, k1, a0, b0);
    threefry2x32(k0, k1, a1, b1);
    rng[0] = a0; rng[1] = a1; key[0] = b0; key[1] = b1;
  }
}

// Y <- shift(Y) = u2node(roll(node2u(Y), -1), last row 0)  (dial_core.py:160-165) as one constant
// (Hn+1)x(Hn+1) matrix; one thread per output element, one CTA per instance
__global__ void mpc_shift_kernel(const float* __restrict__ Msh, const float* __restrict__ Yin,
                                 float* __restrict__ Yout, int n1, int nu) {
  const int i = threadIdx.x;
  Yin += (size_t)blockIdx.x * n1 * nu; Yout += (size_t)blockIdx.x * n1 * nu;
  if (i < n1 * nu) {
    const int k = i / nu, a = i - k * nu;
    float s = 0.f;
    for (int j = 0; j < n1; ++j) s += Msh[k * n1 + j] * Yin[j * nu + a];
    Yout[i] = s;
  }
}

// ---------------------------------------------------------------------------------
// qbar / qdbar / xbar  (core/dial_core.py:133-135): weighted sums over stored trajectories.
// A row of a trajectory array is H * ncol contiguous floats, so out[j] = sum_r w_r traj[r][j] with
// one thread per j reads whole 128-byte lines (consecutive lanes -> consecutive addresses).
//   stage 1: grid (ceil(max_j / 256), TB_CHUNKS row chunks, 3 arrays): per-chunk partials, rows in
//            order, 8 independent loads in flight per thread
//   stage 2: grid H: partials summed in fixed chunk order (bitwise deterministic)
// Batched plans add an instance dimension (stage 1: z = 3 * instance + array, stage 2: y = instance)
// over instance-major trajectories, weights, partials and outputs.  Instance b's trajectories start at
// row b * inst_rows: nrows on a plain plan, K * nrows on an ensemble plan, whose bars read member 0.
// The only bandwidth-shaped kernel of the path: rows * H * (nq + nv + 3 (nbody-1)) * 4 bytes read
// once from L2 / HBM (cfg1: 16 MB, cfg4 shard: 65 MB).
// ---------------------------------------------------------------------------------
#define TB_CHUNKS 32
struct TrajArgs {
  const float* traj[3];
  float* out[3];
  int ncol[3], coloff[3];
  int coltot, nrows, H;
  int inst_rows;   // trajectory rows between two instances (BATCH only)
  const float* weights;
  int w_offset, mean_row, mean_weight_index, include_mean;
  float* partial;  // [TB_CHUNKS][H][coltot]
};

// (32 registers: one CTA fits beside the 448-thread rollout CTA of the next iteration, which the bars overlap)
// BATCH = false (single-instance plans) compiles to the instance-free code: the bars of a plain plan
// pay nothing for the instance dimension.  BATCH only: an instance past its iteration limit at iteration
// `iter` (schedule_runs over iter_lim) keeps its bars.  (Outside TrajArgs: the instance-free code keeps
// its parameter layout.)
template <bool BATCH>
__global__ void __launch_bounds__(256, 8) trajbar_partial_kernel(const TrajArgs T, const int32_t* __restrict__ iter_lim, int iter) {
  const int chunk = blockIdx.y, arr = BATCH ? blockIdx.z % 3 : blockIdx.z, inst = BATCH ? blockIdx.z / 3 : 0;
  const int ncol = arr == 0 ? T.ncol[0] : (arr == 1 ? T.ncol[1] : T.ncol[2]), len = T.H * ncol;
  const int coloff = arr == 0 ? T.coloff[0] : (arr == 1 ? T.coloff[1] : T.coloff[2]);
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (blockIdx.x * 256 >= len || (BATCH && !schedule_runs(iter_lim, inst, iter))) return;
  const float* __restrict__ traj = (arr == 0 ? T.traj[0] : (arr == 1 ? T.traj[1] : T.traj[2])) + (size_t)inst * T.inst_rows * len;
  const float* wts = BATCH ? T.weights + (size_t)inst * (T.mean_weight_index + 1) : T.weights;
  const int per = (T.nrows + TB_CHUNKS - 1) / TB_CHUNKS;
  const int r0 = chunk * per, r1 = min(T.nrows, r0 + per);
  const int jj = j < len ? j : len - 1;
  float a = 0.f;
  for (int r = r0; r < r1; r += 8) {
    float wv[8], xv[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int rr = r + k;
      float wgt = 0.f;
      if (rr < r1) {
        if (rr == T.mean_row) wgt = T.include_mean ? wts[T.mean_weight_index] : 0.f;
        else wgt = wts[T.w_offset + rr];
      }
      wv[k] = wgt;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k)   // weight 0: a diverged sample (NaN trajectory) or a row beyond the chunk: not read
      xv[k] = (wv[k] != 0.f) ? traj[(size_t)(r + k) * len + jj] : 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) a += wv[k] * xv[k];
  }
  if (j < len) {
    const int t = j / ncol, c = j - t * ncol;
    T.partial[(((size_t)inst * TB_CHUNKS + chunk) * T.H + t) * T.coltot + coloff + c] = a;
  }
}

template <bool BATCH>
__global__ void __launch_bounds__(128, 8) trajbar_final_kernel(const TrajArgs T, const int32_t* __restrict__ iter_lim, int iter) {
  const int t = blockIdx.x, inst = BATCH ? blockIdx.y : 0;
  if (BATCH && !schedule_runs(iter_lim, inst, iter)) return;
  const float* partial = T.partial + (size_t)inst * TB_CHUNKS * T.H * T.coltot;
  for (int col = threadIdx.x; col < T.coltot; col += blockDim.x) {
    float s = 0.f;
#pragma unroll 8
    for (int ch = 0; ch < TB_CHUNKS; ++ch) s += partial[((size_t)ch * T.H + t) * T.coltot + col];
    float* out; int ncol, off;   // (no dynamic indexing of the kernel parameter: it would be copied to the stack)
    if (col >= T.coloff[2]) { out = T.out[2]; ncol = T.ncol[2]; off = T.coloff[2]; }
    else if (col >= T.coloff[1]) { out = T.out[1]; ncol = T.ncol[1]; off = T.coloff[1]; }
    else { out = T.out[0]; ncol = T.ncol[0]; off = T.coloff[0]; }
    if (out) out[((size_t)inst * T.H + t) * ncol + (col - off)] = s;
  }
}

// Ensemble plans (n_ens = K >= 2): rews[b][i] = instance b's risk measure risk[b] of the member rewards
// r[b][0..K-1][i] (ens_risk_reduce; the mean: (((r0 + r1) + ...) + r_{K-1}) / K), fp32 with
// round-to-nearest (the library is built with -use_fast_math, whose `/` is approximate).  One thread per
// (instance, sample); grid.y is the instance, so a CTA reads one setting and takes one branch.  An
// instance adapting to its plant (adapt[b].on) takes the belief-weighted branch of its measure
// (ens_risk_reduce_weighted) over its belief w [B][K].
__global__ void __launch_bounds__(256) ensemble_reduce_kernel(const float* __restrict__ r, const EnsRisk* __restrict__ risk,
                                                              const EnsAdapt* __restrict__ adapt, const float* __restrict__ belief,
                                                              int K, int n1, float* __restrict__ rews,
                                                              const int32_t* __restrict__ iter_lim, int iter) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= n1 || !schedule_runs(iter_lim, b, iter)) return;   // a skipped instance keeps its scores
  const EnsRisk R = risk[b];
  const float* rb = r + (size_t)b * K * n1 + i;
  rews[(size_t)b * n1 + i] = adapt[b].on ? ens_risk_reduce_weighted(rb, (size_t)n1, K, R, belief + (size_t)b * K, adapt[b].prune)
                                         : ens_risk_reduce(rb, (size_t)n1, K, R);
}

// Ensemble adaptation, before the plant's env step: us [B K][nu] row b K + k = Y[b][0], the action of
// instance b, so that the member-prediction launch reads its action at the rollout kernel's row stride.
__global__ void __launch_bounds__(128) ens_gather_kernel(const float* __restrict__ Y, int K, int n1, int nu,
                                                         float* __restrict__ us) {
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < K * nu; i += blockDim.x) us[(size_t)b * K * nu + i] = Y[(size_t)b * n1 * nu + i % nu];
}

// Ensemble adaptation, after the plant's env step: one warp per instance.  Lane k < K scores member k's
// predicted qvel vhat [B K][nv] against the observed qvel [B][nv] (ens_member_loglik); lane 0 then
// updates the belief L / w [B][K] in member order (ens_belief_update).  ell [B][K] keeps the last l.
// Instances that do not adapt are left as they are.
__global__ void __launch_bounds__(32) ens_belief_kernel(const float* __restrict__ vhat, const float* __restrict__ qvel,
                                                        const EnsAdapt* __restrict__ adapt, int K, int nv,
                                                        double* __restrict__ L, float* __restrict__ w, float* __restrict__ ell) {
  const int b = blockIdx.x, lane = threadIdx.x;
  if (!adapt[b].on) return;
  __shared__ double l[DIAL_MAXENS];
  if (lane < K) {
    l[lane] = ens_member_loglik(vhat + ((size_t)b * K + lane) * nv, qvel + (size_t)b * nv, adapt[b].sigma, nv);
    ell[(size_t)b * K + lane] = (float)l[lane];
  }
  __syncwarp();
  if (lane == 0) ens_belief_update(L + (size_t)b * K, w + (size_t)b * K, l, K, (double)adapt[b].forget);
}

// Control latency (dial_plan_set_instance_delay), one CTA per instance b: its queue's step
// (delay_queue_step; pop in a step with an env step) from its action Y[b][0], the action its env step
// applies (applied [B][nu]), its queue in application order (pending [B][DIAL_MAXDELAY][nu]) and its
// prediction length pred_len[b] (d when it predicts, else 0) for the prediction launches.
__global__ void __launch_bounds__(128) delay_queue_kernel(const DelaySetting* __restrict__ set, int32_t* __restrict__ head,
                                                          float* __restrict__ ring, const float* __restrict__ Y, int n1,
                                                          int nu, int pop, float* __restrict__ applied,
                                                          float* __restrict__ pending, int32_t* __restrict__ pred_len) {
  const int b = blockIdx.x;
  const DelaySetting s = set[b];
  const int h = head[b];
  const size_t q = (size_t)b * DIAL_MAXDELAY * nu;
  const int h1 = delay_queue_step(ring + q, h, s.d, nu, Y + (size_t)b * n1 * nu, applied + (size_t)b * nu, pending + q,
                                  pop != 0, threadIdx.x, blockDim.x);
  __syncthreads();   // every thread has read head[b]
  if (threadIdx.x == 0) { head[b] = h1; pred_len[b] = s.predict && s.d > 0 ? s.d : 0; }
}

// dial_plan_set_instance_delay: instance b's queue refilled with d copies of Y[b][0], front at slot 0, and
// its pending rows laid out (one CTA)
__global__ void __launch_bounds__(128) delay_refill_kernel(int b, int d, int32_t* __restrict__ head, float* __restrict__ ring,
                                                           const float* __restrict__ Y, int n1, int nu,
                                                           float* __restrict__ pending) {
  const size_t q = (size_t)b * DIAL_MAXDELAY * nu;
  const float* y0 = Y + (size_t)b * n1 * nu;
  for (int a = threadIdx.x; a < nu; a += blockDim.x)
    for (int j = 0; j < d; ++j) ring[q + (size_t)j * nu + a] = y0[a];
  delay_queue_step(ring + q, 0, d, nu, y0, nullptr, pending + q, false, threadIdx.x, blockDim.x);
  if (threadIdx.x == 0) head[b] = 0;
}

// The buffers of the observation (dial_plan_set_instance_observation), instance-major: the rings [B], their
// records [B][DIAL_OBSRING][*], the observation [B][*] and its age [B], the prediction's actions
// [B][DIAL_MAXDELAY][nu] and lengths [B].
struct ObsBuffers {
  ObsRing* ring;
  float *rq, *rv, *rw, *ra;
  int32_t* rc;
  float *oq, *ov, *ow;
  int32_t *oc, *age;
  float* seq;
  int32_t* len;
};

// Observation, one CTA per instance b, after the plant's env step and the shift: its ring's step (a record
// pushed in a step with an env step, seeded after a reset; observe_advance / observe_record), its observation
// (observe_emit) into the observed state and the planning state (pq.. [B][*]), the prediction's actions and
// the prediction length (age + d_b when b predicts through its delay setting `dset`, else 0).  `act`: the
// actions the env step applied, one row of act_row floats per instance.
__global__ void __launch_bounds__(128) observe_kernel(const DevModel* __restrict__ M, const ObsSetting* __restrict__ set,
                                                      ObsBuffers O, const DelaySetting* __restrict__ dset,
                                                      const float* __restrict__ pending, int env_step,
                                                      const float* __restrict__ qpos, const float* __restrict__ qvel,
                                                      const float* __restrict__ warm, const int32_t* __restrict__ cnt,
                                                      const float* __restrict__ act, int act_row, float* __restrict__ pq,
                                                      float* __restrict__ pv, float* __restrict__ pw, int32_t* __restrict__ pc) {
  const int b = blockIdx.x;
  const dial_model_desc& m = M->m;
  const size_t nq = m.nq, nv = m.nv, nu = m.nu, R = DIAL_OBSRING;
  const ObsSetting& s = set[b];
  const ObsRing r = O.ring[b];
  const DelaySetting ds = dset ? dset[b] : DelaySetting{0, 0};
  const ObsRing r1 = observe_advance(s, r, env_step != 0);
  ObsView V;
  V.qpos = qpos + b * nq; V.qvel = qvel + b * nv; V.warm = warm + b * nv; V.cnt = cnt + 2 * b;
  V.act = env_step ? act + b * act_row : nullptr;
  V.rq = O.rq + b * R * nq; V.rv = O.rv + b * R * nv; V.rw = O.rw + b * R * nv; V.ra = O.ra + b * R * nu;
  V.rc = O.rc + b * R * 2;
  V.oq = O.oq + b * nq; V.ov = O.ov + b * nv; V.ow = O.ow + b * nv; V.oc = O.oc + 2 * b;
  V.pq = pq + b * nq; V.pv = pv + b * nv; V.pw = pw + b * nv; V.pc = pc + 2 * b;
  V.seq = O.seq + b * DIAL_MAXDELAY * nu;
  V.pending = pending ? pending + b * DIAL_MAXDELAY * nu : nullptr;
  observe_record(observe_pushes(s, r, env_step != 0), r1, V, (int)nq, (int)nv, (int)nu, threadIdx.x, blockDim.x);
  __syncthreads();   // the new record is complete, and every thread has read ring[b]
  observe_emit(s, r1, m, ds.d, V, threadIdx.x, blockDim.x);
  if (threadIdx.x == 0) {
    const int age = observe_age(s, r1);
    O.ring[b] = r1; O.age[b] = age; O.len[b] = ds.predict ? age + ds.d : 0;
  }
}

// dial_plan_set_instance_observation: instance b's ring reset (the next observe step seeds it), its noise
// key that of its setting
__global__ void observe_reset_kernel(int b, const ObsSetting* __restrict__ set, ObsRing* __restrict__ ring) {
  ObsRing r;
  r.head = 0; r.count = 0;
  r.key[0] = set[b].key[0]; r.key[1] = set[b].key[1]; r.sub[0] = 0u; r.sub[1] = 0u;
  ring[b] = r;
}

// Pushes (dial_plan_set_instance_pushes), one warp per instance b, after the plant's env step and adaptation's
// belief update: when some entry of its table T[b] fires at its post-step counter, its plant qvel takes the
// impulse response M^-1 J^T [torque; force] dt in fp64 on its plant model (models[b], else the plan's model M0):
// push_kinematics on lane 0, the mass-matrix rows and the generalized impulse on every lane, the Cholesky solve
// on lane 0.  An instance with no entry firing leaves at entry.
__global__ void __launch_bounds__(32) push_kernel(const DevModel* __restrict__ M0, const DevModel* __restrict__ models,
                                                  const PushTable* __restrict__ T, const int32_t* __restrict__ cnt,
                                                  const float* __restrict__ qpos, float* __restrict__ qvel, double dt) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int step = cnt[2 * b];
  if (!push_any(T[b], step)) return;
  __shared__ PushWork W;
  const DevModel& D = models ? models[b] : *M0;
  const int nq = D.m.nq, nv = D.m.nv;
  if (lane == 0) push_kinematics(D.m, qpos + (size_t)b * nq, W);
  __syncwarp();
  push_rows(D, T[b], step, dt, W, lane, 32);
  __syncwarp();
  if (lane == 0) push_solve(nv, W);
  __syncwarp();
  for (int i = lane; i < nv; i += 32) qvel[(size_t)b * nv + i] = push_add(qvel[(size_t)b * nv + i], W.g[i]);
}

// ---------------------------------------------------------------------------------
// plan object
// ---------------------------------------------------------------------------------
// A per-instance setting the captured graphs read between replays: the device array of n slots of `width`
// elements, its pinned host staging and, per slot, the event of the last copy out of the staging slot.
// `d` stays null until allocate(): the plan's launch key (launch_key) tells an unset setting by it.
template <class T> struct Staged {
  T* d = nullptr;
  T* h = nullptr;
  size_t width = 1;
  std::vector<cudaEvent_t> ev;
  // every element starts as `init`, uploaded synchronously; on failure nothing stays allocated
  cudaError_t allocate(size_t n, size_t w, const T& init) {
    width = w;
    cudaError_t e = cudaMallocHost(&h, n * w * sizeof(T));
    if (e == cudaSuccess) e = cudaMalloc(&d, n * w * sizeof(T));
    if (e == cudaSuccess) {
      for (size_t i = 0; i < n * w; ++i) h[i] = init;
      e = cudaMemcpy(d, h, n * w * sizeof(T), cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) { release(); return e; }
    ev.assign(n, nullptr);
    return cudaSuccess;
  }
  // `fill(h_slot)` rewrites slot `s` of the staging, once the previous copy out of it has run; the slot is
  // then copied stream-ordered on `st`, and the captured graphs read it at their next replay
  template <class F> cudaError_t put(size_t s, F fill, cudaStream_t st) {
    cudaEvent_t& e_s = ev[s];
    cudaError_t e = e_s ? cudaEventSynchronize(e_s) : cudaEventCreateWithFlags(&e_s, cudaEventDisableTiming);
    if (e == cudaSuccess) {
      fill(h + s * width);
      e = cudaMemcpyAsync(d + s * width, h + s * width, width * sizeof(T), cudaMemcpyHostToDevice, st);
    }
    if (e == cudaSuccess) e = cudaEventRecord(e_s, st);
    return e;
  }
  void release() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    ev.clear();
    cudaFree(d); cudaFreeHost(h);
    d = nullptr; h = nullptr;
  }
};

// The host-side facts mpc_enqueue branches on or bakes into a capture, all derived from the plan's settings
// (launch_key): which optional buffers are allocated (an allocation lasts as long as the plan), whether some
// instance predicts through its action delay, and the number of prediction launches.  A captured
// control-step graph replays what mpc_enqueue enqueues under the key it was captured with.
struct LaunchKey {
  bool models = false, members = false, sched = false, lims = false, adapt = false, delay = false, obs = false;
  bool push = false;       // some instance was given a push table: the push launch runs after every env step
  bool plant = false;      // some instance was given a plant fidelity: the plant's env step runs on the plant slots
  uint32_t plant_ks = 0;   // the distinct substep counts in use (bit k - 1: substeps k), one plant launch each
  bool terrain[2] = {false, false};   // some instance was given a terrain on side DIAL_TERRAIN_PLANT / _PLANNER:
                                      // that side's launches read the terrain table, in the terrain build
  bool predicts = false;   // some instance predicts through a delay d_b > 0: the queue launch also runs without an env step
  int npred = 0;           // prediction launches
  // the planner's rollouts start from the planning state, not the plant state
  bool planning() const { return obs || npred > 0; }
  bool operator!=(const LaunchKey& o) const {
    return models != o.models || members != o.members || sched != o.sched || lims != o.lims || adapt != o.adapt ||
           delay != o.delay || obs != o.obs || push != o.push || plant != o.plant || plant_ks != o.plant_ks ||
           predicts != o.predicts || npred != o.npred || terrain[0] != o.terrain[0] || terrain[1] != o.terrain[1];
  }
};

struct dial_plan {
  DevModel hM;
  DevPlan hP;
  DevModel* dM = nullptr;
  DevPlan* dP = nullptr;
  int variant = 0;
  // the rollout launchers (resolve_kernels): `flat` serves the launches without a terrain, `generic` those on
  // the plant's plan descriptors, `terrain` (null: none) those that read a terrain table; `name` names `flat`
  struct { dial_launch_fn flat, generic, terrain; const char* name; } kernels{};
  // lock-step level of a launch of 2 or more warps per CTA (RolloutArgs.lockstep): a CTA barrier per env step
  // shares the instruction fetch on every path; the generic tree adds one before the constraint solve, and the
  // dense path, whose unrolled solver is hundreds of KB of SASS, one per Newton iteration
  int lockstep = 1;
  int n_inst = 1;               // independent planner instances (dial_plan_desc.n_inst)
  int n_ens = 0;                // planning models per instance (dial_plan_desc.n_ens)
  int num_sms = 132;
  size_t smem_bytes = 0;
  // workspaces
  // trajectory workspaces [n_inst, max(n_ens, 1), Nsample+1, Hs+1, *], double-buffered so that the bars
  // of iteration i (side stream) can overlap the rollout of iteration i+1
  float *traj_q[2] = {nullptr, nullptr}, *traj_qd[2] = {nullptr, nullptr}, *traj_x[2] = {nullptr, nullptr};
  int cur = 0;
  float* weights = nullptr;                                        // [Ntotal+1]
  float* weights2 = nullptr;                                       // second buffer: the bars of iteration i overlap iteration i+1
  cudaStream_t side = nullptr;                                     // bars branch of the control-step graph
  cudaEvent_t ev_main[2] = {nullptr, nullptr}, ev_side[2] = {nullptr, nullptr};
  float* partial = nullptr;
  float* tb_partial = nullptr;
  unsigned int* counter = nullptr;
  float* zeros = nullptr;                                          // [nv]
  int ybar_grid = 0;
  int upd_grid = 0;             // grid of the fused update kernel: about 8 samples per thread slot
  int64_t launches = 0;
  float* dbg = nullptr;  // optional device counters (DIAL_DEBUG_COUNTERS=1)
  // device-resident MPC loop
  dial_mpc_buffers mpc{};       // caller-owned state block (dial_mpc_bind)
  bool mpc_bound = false;
  float* mpc_Msh = nullptr;     // [Hn+1][Hn+1] shift matrix
  float* mpc_Y1 = nullptr;      // ping-pong partner of mpc.Y
  uint32_t* mpc_key = nullptr;  // sampling key of the current reverse_once
  struct MpcGraph { int n_diffuse, env_step, seen; cudaGraphExec_t exec; int64_t launches; };
  std::vector<MpcGraph> mpc_graphs;
  // the launch key of the current settings, refreshed by every setter that changes one; and that of the last
  // dial_mpc_step, under which every graph in mpc_graphs was captured
  LaunchKey key, ran;
  // per-instance models (dial_plan_set_instance_model): [n_inst] slots read by dial_mpc_step, allocated by
  // the first call
  Staged<DevModel> models;
  // ensemble members (dial_plan_set_ensemble_model): the same for [n_inst * n_ens] member slots, and the
  // members' rewards [n_inst, n_ens, Nsample+1] of one reverse_once (n_ens >= 2)
  Staged<DevModel> members;
  float* ens_rews = nullptr;
  // risk measure per instance (dial_plan_set_ensemble_risk, n_ens >= 2): [n_inst] slots read by the reduction
  Staged<EnsRisk> risk;
  // adaptation to the plant (dial_plan_set_ensemble_adapt / _belief, n_ens >= 2): the settings [n_inst]; the
  // belief L [n_inst, n_ens] in fp64 and w in fp32, one slot of n_ens per instance; the last update's l in
  // fp32.  pred_us [n_inst n_ens, nu] / pred_qd [n_inst n_ens, nv] (the members' predictions) are
  // allocated by the first call that turns adaptation on; until then the graphs hold no adaptation launch.
  Staged<EnsAdapt> adapt;
  Staged<double> belief_L;
  Staged<float> belief_w;
  float* dEll = nullptr;
  float* pred_us = nullptr;
  float* pred_qd = nullptr;
  // per-instance sampling schedules (dial_plan_set_instance_schedule): [n_inst] slots; and the iteration
  // limits (dial_plan_set_instance_iterations): one slot of n_inst counts.  Each is allocated by its first
  // call; the staging `h` mirrors what the device holds
  Staged<InstSchedule> sched;
  Staged<int32_t> lims;
  // the planning state the planner's rollouts start from once some instance predicts or observes (qpos, qvel,
  // warm start, counters [n_inst][*]) and, on an ensemble plan, the planning models [n_inst] (a copy of member
  // (b, 0)); allocated by whichever of dial_plan_set_instance_delay and _observation runs first
  struct PlanningState {
    float *qpos = nullptr, *qvel = nullptr, *warm = nullptr;
    int32_t* cnt = nullptr;
    DevModel* models = nullptr;
  } planning;
  // per-instance control latency (dial_plan_set_instance_delay): the settings [n_inst] (the staging mirrors
  // the device), and, allocated with them, the queues
  Staged<DelaySetting> delay;
  // the queues: front slots [n_inst] and rings [n_inst][DIAL_MAXDELAY][nu], the applied actions [n_inst][nu],
  // the queues in application order [n_inst][DIAL_MAXDELAY][nu] and the prediction lengths [n_inst]
  struct DelayQueue {
    int32_t* head = nullptr;
    float *ring = nullptr, *applied = nullptr, *pending = nullptr;
    int32_t* len = nullptr;
  } queue;
  // per-instance observation (dial_plan_set_instance_observation): the settings [n_inst] (the staging mirrors
  // the device) and, allocated with them by the first call, the rings and observations
  Staged<ObsSetting> obs;
  ObsBuffers ob{};
  // per-instance push tables (dial_plan_set_instance_pushes): [n_inst] slots (the staging mirrors the device),
  // allocated by the first table set
  Staged<PushTable> pushes;
  // per-instance plant fidelity (dial_plan_set_instance_plant), allocated by the first setting: the settings
  // [n_inst] (host only, substeps 0: none); the plant model slots [n_inst] (instance b's model, models[b] or the
  // plan's, with its setting's timestep / k and solver settings); the plan descriptors of the plant, slot k - 1
  // with n_frames = k * n_frames (refreshed while k is in use); and per substep count k the 0/1 mask [n_inst]
  // of the instances in its group, slot k - 1 (the iteration limits of its launch)
  std::vector<dial_plant> plant;
  Staged<DevModel> plant_models;
  Staged<DevPlan> plant_plans;
  Staged<int32_t> plant_mask;
  // per-instance terrain (dial_plan_set_instance_terrain), per side, allocated by the first terrain on that side:
  // the descriptors [n_inst] (nx 0: flat) and each instance's heights, one slot as wide as the largest table
  // it was given so far
  Staged<DevTerrain> terrain[2];
  std::vector<Staged<float>> heights[2];
  // the plan's device buffers that cudaMalloc allocated, by the address of the pointer holding each (own)
  std::vector<void**> owned;
  // cudaMalloc `bytes` into `ptr`, which the plan owns from then on (free_since, dial_plan_destroy); with
  // `zero`, also cleared stream-ordered on `st`.  Does nothing once `e` holds an error, so a group of calls
  // checks it once.
  template <class T> cudaError_t own(cudaError_t& e, T*& ptr, size_t bytes, bool zero = false, cudaStream_t st = nullptr) {
    void** slot = reinterpret_cast<void**>(&ptr);
    if (e == cudaSuccess && (e = cudaMalloc(slot, bytes)) == cudaSuccess) owned.push_back(slot);
    if (e == cudaSuccess && zero) e = cudaMemsetAsync(ptr, 0, bytes, st);
    return e;
  }
  // frees the buffers owned since owned.size() was `mark`, and nulls their pointers
  void free_since(size_t mark) {
    for (; owned.size() > mark; owned.pop_back()) { cudaFree(*owned.back()); *owned.back() = nullptr; }
  }
  // multi-GPU exchange over NVLink peer memory (dial_exchange_*): one cudaMalloc per rank, mapped
  // into every peer with CUDA IPC.  Word offsets inside the block are the same on every rank.
  struct Exchange {
    bool on = false;
    int rank = 0, world = 1, nbar = 0;
    uint32_t* base[DIAL_MAXRANK] = {nullptr};   // base[rank] = own allocation, others = IPC mappings
    size_t words = 0, o_mbox = 0, o_bars = 0, o_flags = 0, o_bflags = 0, o_local = 0;
    float* bars_partial = nullptr;              // local staging of this rank's partial bars [nbar]
    float* mbox(int p) const { return reinterpret_cast<float*>(base[p] + o_mbox); }
    float* bars(int p) const { return reinterpret_cast<float*>(base[p] + o_bars); }
    uint32_t* flags(int p) const { return base[p] + o_flags; }
    uint32_t* bflags(int p) const { return base[p] + o_bflags; }
    uint32_t* seq() const { return base[rank] + o_local; }
    unsigned int* done() const { return base[rank] + o_local + 1; }
    uint32_t* err() const { return base[rank] + o_local + 2; }
    uint32_t* bseq() const { return base[rank] + o_local + 3; }
  } xch;
};

// the control-step graphs captured so far: dial_mpc_step captures them again on their next use
static void drop_graphs(dial_plan* p) {
  for (auto& g : p->mpc_graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  p->mpc_graphs.clear();
}

// instance b's plant substep count: its setting's, or 1 without one
static int plant_substeps(const dial_plan* p, int b) {
  return p->plant.empty() || p->plant[b].substeps == 0 ? 1 : p->plant[b].substeps;
}

// The launch key of the plan's current settings (the staging mirrors the device).  The prediction runs
// max(k_b + d_b) launches over the predicting instances, k_b the observation delay of an observing instance
// while the observe launch runs, else 0.
static LaunchKey launch_key(const dial_plan* p) {
  LaunchKey k;
  k.models = p->models.d != nullptr; k.members = p->members.d != nullptr;
  k.sched = p->sched.d != nullptr; k.lims = p->lims.d != nullptr; k.adapt = p->pred_qd != nullptr;
  k.delay = p->delay.d != nullptr; k.obs = p->obs.d != nullptr; k.push = p->pushes.d != nullptr;
  k.plant = p->plant_models.d != nullptr;
  k.terrain[0] = p->terrain[0].d != nullptr; k.terrain[1] = p->terrain[1].d != nullptr;
  for (int b = 0; k.plant && b < p->n_inst; ++b) k.plant_ks |= 1u << (plant_substeps(p, b) - 1);
  for (int b = 0; k.delay && b < p->n_inst; ++b) {
    const DelaySetting& s = p->delay.h[b];
    const int n = s.d + (k.obs && p->obs.h[b].on ? p->obs.h[b].k : 0);
    if (!s.predict) continue;
    k.predicts |= s.d > 0;
    k.npred = n > k.npred ? n : k.npred;
  }
  return k;
}

static void fill_xch(const dial_plan* p, RolloutArgs& A) {
  if (!p->xch.on) return;
  A.xch_world = p->xch.world; A.xch_rank = p->xch.rank;
  for (int r = 0; r < p->xch.world; ++r) { A.xch_mbox[r] = p->xch.mbox(r); A.xch_flags[r] = p->xch.flags(r); }
  A.xch_seq = p->xch.seq(); A.xch_done = p->xch.done();
}
static XchWait xch_wait_args(const dial_plan* p, float* rews_copy) {
  XchWait X; memset(&X, 0, sizeof(X));
  if (p->xch.on) {
    X.mbox = p->xch.mbox(p->xch.rank); X.flags = p->xch.flags(p->xch.rank); X.seq = p->xch.seq(); X.err = p->xch.err();
    X.rews_copy = rews_copy; X.world = p->xch.world;
  }
  return X;
}

extern "C" int dial_abi_version(void) { return DIAL_ABI_VERSION; }
extern "C" const char* dial_last_error(void) { return g_err.c_str(); }
extern "C" size_t dial_sizeof(int which) {
  return which == 0 ? sizeof(dial_model_desc) : which == 1 ? sizeof(dial_plan_desc) : which == 2 ? sizeof(dial_state)
       : which == 3 ? sizeof(dial_mpc_buffers) : which == 4 ? sizeof(dial_task) : which == 5 ? sizeof(dial_push)
       : which == 6 ? sizeof(dial_plant) : which == 7 ? sizeof(dial_terrain) : 0;
}

// The plan's rollout launchers, fixed by its model, variant and plan descriptor.  Solver instantiation by tree
// shape: star<3,6> (quadruped), star<5,7> (humanoid), star<5,6>, dense<22> (elliptic cones), generic tree.
// `flat` is the shape-specialised kernel of the variant when one matches (not with DIAL_FORCE_GENERIC_SHAPE=1:
// it computes bit for bit what the generic one does, and tests compare the two), else the variant's.
static void resolve_kernels(dial_plan* p) {
  static const char* const names[] = {"v0", "v1", "v2", "v3", "v4"};
  p->kernels.name = names[p->variant];
#ifdef DIAL_ONLY_VARIANT
  p->kernels.flat = p->kernels.generic = DIAL_V_LAUNCHER;   // the variant was checked against DIAL_ONLY_VARIANT
#ifdef DIAL_TERRAIN
  p->kernels.terrain = DIAL_V_LAUNCHER;
#endif
#else
  static const dial_launch_fn generic[] = {dial_launch_rollout_v0, dial_launch_rollout_v1, dial_launch_rollout_v2,
                                           dial_launch_rollout_v3, dial_launch_rollout_v4};
  static const dial_launch_fn terrain[] = {dial_launch_rollout_v0_terrain, dial_launch_rollout_v1_terrain,
                                           dial_launch_rollout_v2_terrain, nullptr, dial_launch_rollout_v4_terrain};
  p->kernels.flat = p->kernels.generic = generic[p->variant];
  p->kernels.terrain = terrain[p->variant];
  if (p->variant == 1 && !getenv("DIAL_FORCE_GENERIC_SHAPE"))
    for (const auto& s : kShapes)
      if (s.matches(p->hM, p->hP.c)) { p->kernels.flat = s.launch; p->kernels.name = s.name; break; }
#endif
}

// One rollout launch of `wpc` warps per CTA (1..16; one kernel serves all).  `dP`: the plan descriptor the
// launch reads (null: the plan's own); `generic`: the generic kernel of the plan's variant even where a
// shape-specialised one matches (whose solver counts and n_frames are fixed).
static cudaError_t launch_rollout(dial_plan* p, const RolloutArgs& A, int wpc, cudaStream_t st,
                                  const DevPlan* dP = nullptr, bool generic = false) {
  const size_t smem = sizeof(DevModel) + sizeof(DevPlan) + (size_t)wpc * p->hM.warp_floats * sizeof(float);
  p->launches++;
  const dial_launch_fn launch = A.terrain ? p->kernels.terrain : generic ? p->kernels.generic : p->kernels.flat;
  if (!launch) return cudaErrorInvalidDeviceFunction;
  return launch(p->dM, dP ? dP : p->dP, A, rollout_grid(A, wpc), wpc, smem, st);
}

// Launch shape.  One CTA per SM with up to 16 warps that re-converge at every env step
// ("lock-step"): the warps of an SM then walk the ~230 KB of straight-line kernel code together
// and share instruction fetches (faster than independent 4-warp CTAs).
static int default_wpc(const dial_plan* p, int nrows) {
  // one CTA per SM holding that SM's share of the rows (any warp count 1..16: the kernel is
  // not specialised on it)
  const int per_sm = (nrows + p->num_sms - 1) / p->num_sms;
  // at most the kernel's __launch_bounds__ (dial_host.h) and what the 227 KB of shared memory of
  // one CTA holds
  const size_t fixed = sizeof(DevModel) + sizeof(DevPlan), slab = (size_t)p->hM.warp_floats * sizeof(float);
  int maxw = DIAL_MAXTHREADS / 32;
  while (maxw > 1 && fixed + maxw * slab > 227 * 1024) --maxw;
  if (per_sm <= maxw) return per_sm;
  // more than one wave of rows: balance the waves of one CTA per SM (balanced waves beat full
  // waves with a ragged last one, and two resident half-size CTAs)
  const int waves = (per_sm + maxw - 1) / maxw;
  return (per_sm + waves - 1) / waves;
}

static cudaError_t launch_rollout_any(dial_plan* p, const RolloutArgs& A0, cudaStream_t st) {
  RolloutArgs A = A0;
  const char* f = getenv("DIAL_WPC");
  int wpc = f ? atoi(f) : 0;
  if (wpc == 0) {
    wpc = default_wpc(p, A.nrows);
    // per-instance or member models: a CTA holds rows of one model slot; spread each slot's rows evenly
    // over the CTAs it needs at that width
    if (A.models && model_rows(A) > 0) {
      const int cpi = (model_rows(A) + wpc - 1) / wpc;
      wpc = (model_rows(A) + cpi - 1) / cpi;
    }
  }
  if (wpc < 1 || wpc > DIAL_MAXTHREADS / 32) return cudaErrorInvalidValue;
  // sync_every (0) and row_counter (null) stay unset: a barrier at every env step, and every warp on its own row
  A.lockstep = wpc >= 2 ? p->lockstep : 0;
  return launch_rollout(p, A, wpc, st);
}

extern "C" dial_plan* dial_plan_create(const dial_model_desc* model, const dial_plan_desc* cfg) {
  if (!model || !cfg) { g_err = "null descriptor"; return nullptr; }
  dial_plan* p = new (std::nothrow) dial_plan();
  if (!p) { g_err = "out of memory"; return nullptr; }
  std::string err;
  if (!derive_model(*model, p->hM, err)) { g_err = err; delete p; return nullptr; }
  {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0)
      p->num_sms = sms;
  }
  p->variant = (getenv("DIAL_FORCE_GENERIC_TREE") && !p->hM.dense) ? 0 : star_variant(p->hM);
  if (p->variant < 0) { g_err = "this build instantiates the dense (elliptic) solver path for nv = " DIAL_STR(DIAL_DENSE_NV) " only (custom builds: dial_mpc_b200.custom compiles it for the model's nv)"; delete p; return nullptr; }
  memset(&p->hP, 0, sizeof(DevPlan));
  p->hP.c = *cfg;
  p->hP.c.cmd_step = -1;      // command overrides come through dial_plan_set_command only
  const dial_plan_desc& c = *cfg;
  if (c.Hsample + 1 > DIAL_MAXH || c.Hnode + 1 > DIAL_MAXNODE || c.Hnode < 1 || c.Nsample < 1 || c.Ntotal < c.Nsample ||
      c.n_frames < 1 || (c.Hnode + 1) * model->nu > YBAR_THREADS || c.n_stage > DIAL_MAXSTAGE) {
    g_err = "invalid plan configuration (Hsample/Hnode/Nsample/n_frames out of range)";
    delete p;
    return nullptr;
  }
  if (c.env_id < DIAL_ENV_GO2_WALK || c.env_id > DIAL_ENV_CUSTOM) { g_err = "unknown env_id"; delete p; return nullptr; }
#ifndef DIAL_CUSTOM_REWARD_FILE
  if (c.env_id == DIAL_ENV_CUSTOM) {
    g_err = "env_id DIAL_ENV_CUSTOM needs a library built with a reward source (dial_mpc_b200.custom.build_library); this is the stock build";
    delete p; return nullptr;
  }
#endif
#ifdef DIAL_ONLY_VARIANT
  if (p->variant != DIAL_ONLY_VARIANT) {
    g_err = "this custom build holds solver variant " + std::to_string(DIAL_ONLY_VARIANT) + " only, the model needs " + std::to_string(p->variant);
    delete p; return nullptr;
  }
#endif
  if (c.n_user < 0 || c.n_user > DIAL_MAXUSER) { g_err = "n_user out of range"; delete p; return nullptr; }
  if (c.n_inst < 0) { g_err = "n_inst must be >= 0 (0 or 1: a single instance)"; delete p; return nullptr; }
  if (c.n_inst > 1) {
    if (c.Ntotal != c.Nsample) { g_err = "a batched plan (n_inst > 1) cannot be sharded (Ntotal must equal Nsample)"; delete p; return nullptr; }
    if (c.Nsample + 1 > (1 << 17)) { g_err = "a batched plan (n_inst > 1) needs Nsample + 1 <= 131072 (the fused update)"; delete p; return nullptr; }
    // the instance is grid dimension z / 3 of the bars kernel (<= 65535) and rows are int32
    if (c.n_inst > 65535 / 3 || (int64_t)c.n_inst * (c.Nsample + 1) > 0x7fffffff) {
      g_err = "n_inst too large: at most 21845 instances and 2^31 - 1 rows per rollout launch"; delete p; return nullptr;
    }
  }
  p->n_inst = c.n_inst > 1 ? c.n_inst : 1;
  if (c.n_ens < 0 || c.n_ens > DIAL_MAXENS) { g_err = "n_ens out of range (0..DIAL_MAXENS = " DIAL_STR(DIAL_MAXENS) ")"; delete p; return nullptr; }
  if (c.n_ens >= 1) {
    if (c.Ntotal != c.Nsample) { g_err = "an ensemble plan (n_ens >= 1) cannot be sharded (Ntotal must equal Nsample)"; delete p; return nullptr; }
    if ((int64_t)p->n_inst * c.n_ens * (c.Nsample + 1) > 0x7fffffff) { g_err = "n_inst * n_ens * (Nsample + 1) exceeds 2^31 - 1 rows per rollout launch"; delete p; return nullptr; }
  }
  p->n_ens = c.n_ens;
  resolve_kernels(p);
  p->lockstep = p->hM.dense ? 3 : p->hM.s_on ? 1 : 2;
  auto bad = [&](cudaError_t e, const char* what) {
    g_err = std::string(what) + ": " + cudaGetErrorString(e);
    dial_plan_destroy(p);
    return (dial_plan*)nullptr;
  };
  cudaError_t e = cudaSuccess;
  if (p->own(e, p->dM, sizeof(DevModel)) != cudaSuccess) return bad(e, "cudaMalloc(model)");
  if (p->own(e, p->dP, sizeof(DevPlan)) != cudaSuccess) return bad(e, "cudaMalloc(plan)");
  if ((e = cudaMemcpy(p->dM, &p->hM, sizeof(DevModel), cudaMemcpyHostToDevice)) != cudaSuccess) return bad(e, "cudaMemcpy(model)");
  if ((e = cudaMemcpy(p->dP, &p->hP, sizeof(DevPlan), cudaMemcpyHostToDevice)) != cudaSuccess) return bad(e, "cudaMemcpy(plan)");
  const size_t B = (size_t)p->n_inst, H = (size_t)c.Hsample + 1;
  const size_t rows = B * (p->n_ens > 1 ? (size_t)p->n_ens : 1) * ((size_t)c.Nsample + 1);   // every member's trajectories
  const dial_model_desc& m = *model;
  for (int b = 0; b < 2; ++b) {
    if (p->own(e, p->traj_q[b], rows * H * m.nq * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(traj_q)");
    if (p->own(e, p->traj_qd[b], rows * H * m.nv * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(traj_qd)");
    if (p->own(e, p->traj_x[b], rows * H * 3 * (m.nbody - 1) * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(traj_x)");
  }
  if (p->n_ens > 1) {
    if (p->own(e, p->ens_rews, rows * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(ens_rews)");
    // every instance starts at the mean, no instance adapts, every belief starts uniform
    const size_t K = p->n_ens;
    const double L0 = log(1.0 / p->n_ens);
    if ((e = p->risk.allocate(B, 1, ens_risk_derive(p->n_ens, DIAL_ENS_MEAN, 1.f))) != cudaSuccess) return bad(e, "allocate(risk)");
    if ((e = p->adapt.allocate(B, 1, EnsAdapt{})) != cudaSuccess) return bad(e, "allocate(adapt)");
    if ((e = p->belief_L.allocate(B, K, L0)) != cudaSuccess) return bad(e, "allocate(belief)");
    if ((e = p->belief_w.allocate(B, K, (float)exp(L0))) != cudaSuccess) return bad(e, "allocate(belief)");
    if (p->own(e, p->dEll, B * K * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(belief)");
    if ((e = cudaMemset(p->dEll, 0, B * K * sizeof(float))) != cudaSuccess) return bad(e, "cudaMemset(belief)");
  }
  if (p->own(e, p->weights, B * ((size_t)c.Ntotal + 1) * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(weights)");
  if (p->own(e, p->weights2, B * ((size_t)c.Ntotal + 1) * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(weights2)");
  if ((e = cudaStreamCreateWithFlags(&p->side, cudaStreamNonBlocking)) != cudaSuccess) return bad(e, "cudaStreamCreate(side)");
  for (int i = 0; i < 2; ++i) {
    if ((e = cudaEventCreateWithFlags(&p->ev_main[i], cudaEventDisableTiming)) != cudaSuccess) return bad(e, "cudaEventCreate");
    if ((e = cudaEventCreateWithFlags(&p->ev_side[i], cudaEventDisableTiming)) != cudaSuccess) return bad(e, "cudaEventCreate");
  }
  const int ne = (c.Hnode + 1) * m.nu, slots = YBAR_THREADS / ne;
  int g = (c.Ntotal + 1 + slots - 1) / slots;
  p->ybar_grid = g < 1 ? 1 : (g > 2 * p->num_sms ? 2 * p->num_sms : g);   // two CTAs per SM at most
  {
    int gu = (c.Ntotal + 1 + slots * 8 - 1) / (slots * 8);
    p->upd_grid = gu < 1 ? 1 : (gu > p->ybar_grid ? p->ybar_grid : gu);
  }
  if (p->own(e, p->partial, B * p->ybar_grid * (ne + 1) * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(partial)");
  if (p->own(e, p->tb_partial, B * TB_CHUNKS * H * (m.nq + m.nv + 3 * (m.nbody - 1)) * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(tb_partial)");
  if (p->own(e, p->counter, B * sizeof(unsigned int)) != cudaSuccess) return bad(e, "cudaMalloc(counter)");
  if ((e = cudaMemset(p->counter, 0, B * sizeof(unsigned int))) != cudaSuccess) return bad(e, "cudaMemset(counter)");
  if (getenv("DIAL_DEBUG_COUNTERS")) {
    if (p->own(e, p->dbg, 8 * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(dbg)");
    cudaMemset(p->dbg, 0, 8 * sizeof(float));
  }
  if (p->own(e, p->zeros, DIAL_MAXV * sizeof(float)) != cudaSuccess) return bad(e, "cudaMalloc(zeros)");
  if ((e = cudaMemset(p->zeros, 0, DIAL_MAXV * sizeof(float))) != cudaSuccess) return bad(e, "cudaMemset(zeros)");
  return p;
}

extern "C" void dial_plan_destroy(dial_plan* p) {
  if (!p) return;
  drop_graphs(p);
  for (int r = 0; r < DIAL_MAXRANK; ++r) {
    if (!p->xch.base[r]) continue;
    if (r == p->xch.rank) cudaFree(p->xch.base[r]); else cudaIpcCloseMemHandle(p->xch.base[r]);
  }
  cudaFree(p->xch.bars_partial);
  p->models.release(); p->members.release(); p->risk.release();
  p->adapt.release(); p->belief_L.release(); p->belief_w.release(); p->sched.release(); p->lims.release();
  p->delay.release(); p->obs.release(); p->pushes.release();
  p->plant_models.release(); p->plant_plans.release(); p->plant_mask.release();
  for (int s = 0; s < 2; ++s) {
    p->terrain[s].release();
    for (auto& h : p->heights[s]) h.release();
  }
  for (int i = 0; i < 2; ++i) { if (p->ev_main[i]) cudaEventDestroy(p->ev_main[i]); if (p->ev_side[i]) cudaEventDestroy(p->ev_side[i]); }
  if (p->side) cudaStreamDestroy(p->side);
  p->free_since(0);
  delete p;
}

static void fill_state(RolloutArgs& A, const dial_state* s) {
  A.qpos0 = s->qpos; A.qvel0 = s->qvel; A.warm0 = s->qacc_warmstart; A.step0 = s->step; A.stage0 = s->stage;
}

extern "C" int dial_rollout(dial_plan* p, const dial_state* s, const float* us, int B, int H, float* rewss,
                            float* q, float* qd, float* xpos, void* stream) {
  if (!p || !s || !us || !rewss) return fail("dial_rollout: null argument");
  if (B < 1 || H < 1) return fail("dial_rollout: B and H must be positive");
  RolloutArgs A; memset(&A, 0, sizeof(A));
  fill_state(A, s);
  A.nrows = B; A.H = H; A.mode = 0; A.us = us; A.rewss = rewss; A.q = q; A.qd = qd; A.xpos = xpos;
  CUDA_OK(launch_rollout_any(p, A, (cudaStream_t)stream));
  return 0;
}

// The plant's plan descriptors of the substep counts in `ks` (bit k - 1: k), from the plan's host mirror with
// n_frames = k * n_frames, stream-ordered on `st` (nothing before the first plant setting)
static cudaError_t put_plant_plans(dial_plan* p, uint32_t ks, cudaStream_t st) {
  cudaError_t e = cudaSuccess;
  for (int k = 1; p->plant_plans.d && k <= DIAL_MAXSUBSTEPS && e == cudaSuccess; ++k)
    if ((ks >> (k - 1)) & 1u)
      e = p->plant_plans.put(k - 1, [&](DevPlan* h) { *h = p->hP; h->c.n_frames = k * p->hP.c.n_frames; }, st);
  return e;
}

// Instance b's plant model: its instance model (the staging mirrors the device) or the plan's, with the
// timestep and solver settings of its plant setting
static DevModel plant_model(const dial_plan* p, int b) {
  DevModel D = p->models.d ? p->models.h[b] : p->hM;
  const dial_plant& f = p->plant[b];
  if (f.substeps == 0) return D;
  D.m.timestep = D.m.timestep / (float)f.substeps;
  D.m.iterations = f.iterations; D.m.ls_iterations = f.ls_iterations; D.m.tolerance = f.tolerance;
  return D;
}

extern "C" int dial_plan_set_command(dial_plan* p, int cmd_step, const float* vel, const float* ang, void* stream) {
  if (!p) return fail("dial_plan_set_command: null plan");
  if (cmd_step >= 0 && (!vel || !ang)) return fail("dial_plan_set_command: null command");
  dial_plan_desc& c = p->hP.c;
  c.cmd_step = cmd_step;
  for (int i = 0; i < 3; ++i) { c.cmd_vel[i] = cmd_step >= 0 ? vel[i] : 0.f; c.cmd_ang[i] = cmd_step >= 0 ? ang[i] : 0.f; }
  // 28 bytes from pageable host memory: staged by the driver before the call returns, stream-ordered on the device
  const size_t off = offsetof(dial_plan_desc, cmd_step);
  CUDA_OK(cudaMemcpyAsync((char*)p->dP + off, (const char*)&p->hP.c + off, sizeof(int32_t) + 6 * sizeof(float),
                          cudaMemcpyHostToDevice, (cudaStream_t)stream));
  CUDA_OK(put_plant_plans(p, p->key.plant_ks, (cudaStream_t)stream));
  return 0;
}

extern "C" int dial_plan_set_stages(dial_plan* p, int n_stage, const float* pose_seq, const float* yaw_seq,
                                    const float* contact_targets, const float* contact_radius, void* stream) {
  if (!p) return fail("dial_plan_set_stages: null plan");
  if (n_stage < 1 || n_stage > DIAL_MAXSTAGE) return fail("dial_plan_set_stages: n_stage out of range (1..DIAL_MAXSTAGE)");
  if (!pose_seq || !yaw_seq || !contact_targets || !contact_radius) return fail("dial_plan_set_stages: null table");
  dial_plan_desc& c = p->hP.c;
  c.n_stage = n_stage;
  memset(c.pose_seq, 0, sizeof(c.pose_seq)); memset(c.yaw_seq, 0, sizeof(c.yaw_seq));
  memset(c.contact_targets, 0, sizeof(c.contact_targets)); memset(c.contact_radius, 0, sizeof(c.contact_radius));
  memcpy(c.pose_seq, pose_seq, sizeof(float) * 3 * n_stage);
  memcpy(c.yaw_seq, yaw_seq, sizeof(float) * n_stage);
  memcpy(c.contact_targets, contact_targets, sizeof(float) * 12 * n_stage);
  memcpy(c.contact_radius, contact_radius, sizeof(float) * 4 * n_stage);
  // one stream-ordered copy of [n_stage .. n_user) from the plan's own host mirror (pageable: staged
  // by the driver before the call returns)
  const size_t off = offsetof(dial_plan_desc, n_stage), end = offsetof(dial_plan_desc, n_user);
  CUDA_OK(cudaMemcpyAsync((char*)p->dP + off, (const char*)&p->hP.c + off, end - off, cudaMemcpyHostToDevice,
                          (cudaStream_t)stream));
  CUDA_OK(put_plant_plans(p, p->key.plant_ks, (cudaStream_t)stream));
  return 0;
}

static std::string fmt_g(double x) {
  char buf[64];
  snprintf(buf, sizeof(buf), "%g", x);
  return buf;
}

// The checks the per-instance setters share; `fn` names the public call in errors.  A plan (not null) with
// an ensemble of at least k (1 or 2) members:
static int need_ensemble(const dial_plan* p, const char* fn, int k) {
  if (!p) return fail(std::string(fn) + ": null plan");
  if (p->n_ens >= k) return 0;
  if (k == 1) return fail(std::string(fn) + ": the plan has no ensemble (dial_plan_desc.n_ens = 0)");
  return fail(std::string(fn) + ": the plan needs an ensemble of n_ens >= " + std::to_string(k) + " members, it has " + std::to_string(p->n_ens));
}
// b is an instance of the plan:
static int need_instance(const dial_plan* p, const char* fn, int b) {
  if (b >= 0 && b < p->n_inst) return 0;
  return fail(std::string(fn) + ": instance " + std::to_string(b) + " out of range (0.." + std::to_string(p->n_inst - 1) + ")");
}

// Derive `m`, check it against the plan's model and copy it into slot `slot` of the model slots `a` [n],
// allocating them on first use with every slot holding the plan's own model.  `fn` names the public call
// in errors.
static int set_model_slot(dial_plan* p, const char* fn, Staged<DevModel>& a, size_t n, size_t slot,
                          const dial_model_desc* m, cudaStream_t st) {
  std::unique_ptr<DevModel> D(new (std::nothrow) DevModel());
  if (!D) return fail("out of memory");
  std::string err;
  if (!derive_model(*m, *D, err)) return fail(std::string(fn) + ": " + err);
  if (const char* diff = instance_model_difference(p->hM, *D))
    return fail(std::string(fn) + ": field '" + diff + "' differs from the plan's model "
                "(an instance's model may differ in floats other than timestep, jnt_range and actuator_ctrlrange only)");
  cudaError_t e = cudaSuccess;
  if (!a.d && (e = a.allocate(n, 1, p->hM)) != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  e = a.put(slot, [&](DevModel* h) { *h = *D; }, st);
  p->key = launch_key(p);
  CUDA_OK(e);
  return 0;
}

extern "C" int dial_plan_set_instance_model(dial_plan* p, int b, const dial_model_desc* m, void* stream) {
  static const char* fn = "dial_plan_set_instance_model";
  if (!p || !m) return fail(std::string(fn) + ": null argument");
  if (int rc = need_instance(p, fn, b)) return rc;
  if (p->hP.c.Ntotal != p->hP.c.Nsample) return fail(std::string(fn) + ": sharded plans (Ntotal != Nsample) share one model");
  if (int rc = set_model_slot(p, fn, p->models, (size_t)p->n_inst, (size_t)b, m, (cudaStream_t)stream)) return rc;
  // instance b's plant: the new model with its fidelity kept
  if (p->plant_models.d) {
    cudaError_t e = p->plant_models.put(b, [&](DevModel* h) { *h = plant_model(p, b); }, (cudaStream_t)stream);
    if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  }
  return 0;
}

extern "C" int dial_plan_set_ensemble_model(dial_plan* p, int b, int k, const dial_model_desc* m, void* stream) {
  static const char* fn = "dial_plan_set_ensemble_model";
  if (!p || !m) return fail(std::string(fn) + ": null argument");
  if (int rc = need_ensemble(p, fn, 1)) return rc;
  if (int rc = need_instance(p, fn, b)) return rc;
  if (k < 0 || k >= p->n_ens) return fail(std::string(fn) + ": member " + std::to_string(k) + " out of range (0.." + std::to_string(p->n_ens - 1) + ")");
  const size_t slot = (size_t)b * p->n_ens + k;
  if (int rc = set_model_slot(p, fn, p->members, (size_t)p->n_inst * p->n_ens, slot, m, (cudaStream_t)stream)) return rc;
  // member (b, 0) is instance b's planning model for its prediction through a delay
  if (k == 0 && p->planning.models)
    CUDA_OK(cudaMemcpyAsync(p->planning.models + b, p->members.d + slot, sizeof(DevModel), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

extern "C" int dial_plan_set_ensemble_risk(dial_plan* p, int b, int mode, float alpha, void* stream) {
  static const char* fn = "dial_plan_set_ensemble_risk";
  if (int rc = need_ensemble(p, fn, 1)) return rc;
  if (int rc = need_instance(p, fn, b)) return rc;
  if (mode != DIAL_ENS_MEAN && mode != DIAL_ENS_CVAR)
    return fail(std::string(fn) + ": mode " + std::to_string(mode) + " is neither DIAL_ENS_MEAN (0) nor DIAL_ENS_CVAR (1)");
  if (mode == DIAL_ENS_CVAR && !(alpha > 0.f && alpha <= 1.f))   // also rejects NaN and infinities
    return fail(std::string(fn) + ": alpha must be finite and in (0, 1] for DIAL_ENS_CVAR, got " + fmt_g(alpha));
  if (p->n_ens < 2) return 0;   // one member: every risk measure of one reward is that reward
  cudaError_t e = p->risk.put(b, [&](EnsRisk* r) { *r = ens_risk_derive(p->n_ens, mode, alpha); }, (cudaStream_t)stream);
  if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  return 0;
}

extern "C" int dial_plan_member_rewards(dial_plan* p, float* out, void* stream) {
  static const char* fn = "dial_plan_member_rewards";
  if (!p || !out) return fail(std::string(fn) + ": null argument");
  if (int rc = need_ensemble(p, fn, 1)) return rc;
  if (!p->mpc_bound) return fail(std::string(fn) + ": call dial_mpc_bind first");
  const size_t n = (size_t)p->n_inst * p->n_ens * ((size_t)p->hP.c.Nsample + 1);
  const float* src = p->n_ens > 1 ? p->ens_rews : p->mpc.rews;   // n_ens = 1: the rollout writes rews itself
  CUDA_OK(cudaMemcpyAsync(out, src, n * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

extern "C" int dial_plan_set_ensemble_adapt(dial_plan* p, int b, int on, float forget, float prune, const float* sigma, void* stream) {
  static const char* fn = "dial_plan_set_ensemble_adapt";
  if (int rc = need_ensemble(p, fn, 2)) return rc;
  if (int rc = need_instance(p, fn, b)) return rc;
  if (on != 0 && on != 1) return fail(std::string(fn) + ": on must be 0 or 1, got " + std::to_string(on));
  const int K = p->n_ens, nv = p->hM.m.nv;
  if (on) {   // also rejects NaN and infinities
    if (!(forget > 0.f && forget <= 1.f)) return fail(std::string(fn) + ": forget must be in (0, 1], got " + fmt_g(forget));
    if (!(prune >= 0.f && (double)prune < 1.0 / K))
      return fail(std::string(fn) + ": prune must be in [0, 1/K) = [0, " + fmt_g(1.0 / K) + "), got " + fmt_g(prune));
    if (!sigma) return fail(std::string(fn) + ": null sigma");
    for (int j = 0; j < nv; ++j)
      if (!(sigma[j] > 0.f && sigma[j] <= FLT_MAX))
        return fail(std::string(fn) + ": sigma[" + std::to_string(j) + "] must be finite and > 0, got " + fmt_g(sigma[j]));
  }
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  if (on && !p->pred_qd) {   // first instance to adapt: the prediction workspaces
    const size_t rows = (size_t)p->n_inst * K, mark = p->owned.size();
    p->own(e, p->pred_us, rows * p->hM.m.nu * sizeof(float));
    if (p->own(e, p->pred_qd, rows * nv * sizeof(float)) != cudaSuccess) {
      p->free_since(mark);
      return fail(std::string(fn) + ": " + cudaGetErrorString(e));
    }
  }
  e = p->adapt.put(b, [&](EnsAdapt* a) {   // off: the staged forget, prune and sigma are kept
    a->on = on;
    if (on) {
      a->forget = forget; a->prune = prune;
      for (int j = 0; j < DIAL_MAXV; ++j) a->sigma[j] = j < nv ? sigma[j] : 1.f;
    }
  }, st);
  p->key = launch_key(p);
  if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  return 0;
}

extern "C" int dial_plan_set_ensemble_belief(dial_plan* p, int b, const float* w, void* stream) {
  static const char* fn = "dial_plan_set_ensemble_belief";
  if (int rc = need_ensemble(p, fn, 2)) return rc;
  if (int rc = need_instance(p, fn, b)) return rc;
  if (!w) return fail(std::string(fn) + ": null w");
  const int K = p->n_ens;
  double sum = 0.0;
  for (int k = 0; k < K; ++k) {
    if (!(w[k] >= 0.f && w[k] <= FLT_MAX)) return fail(std::string(fn) + ": w[" + std::to_string(k) + "] must be finite and >= 0, got " + fmt_g(w[k]));
    sum += (double)w[k];
  }
  if (!(sum > 0.0)) return fail(std::string(fn) + ": the weights must have a positive sum");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = p->belief_L.put(b, [&](double* L) {
    for (int k = 0; k < K; ++k) L[k] = w[k] > 0.f ? log((double)w[k] / sum) : -INFINITY;
  }, st);
  const double* L = p->belief_L.h + (size_t)b * K;   // w from the L just staged
  if (e == cudaSuccess) e = p->belief_w.put(b, [&](float* W) {
    for (int k = 0; k < K; ++k) W[k] = (float)exp(L[k]);
  }, st);
  if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  return 0;
}

extern "C" int dial_plan_ensemble_belief(dial_plan* p, float* w, float* loglik, void* stream) {
  if (int rc = need_ensemble(p, "dial_plan_ensemble_belief", 2)) return rc;
  const size_t n = (size_t)p->n_inst * p->n_ens * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  if (w) CUDA_OK(cudaMemcpyAsync(w, p->belief_w.d, n, cudaMemcpyDeviceToDevice, st));
  if (loglik) CUDA_OK(cudaMemcpyAsync(loglik, p->dEll, n, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// The plans the per-instance schedule calls accept: not sharded, within the fused update's size.
static int need_schedulable(const dial_plan* p, const char* fn) {
  const dial_plan_desc& c = p->hP.c;
  if (c.Ntotal != c.Nsample) return fail(std::string(fn) + ": sharded plans (Ntotal != Nsample) share the plan's schedule");
  if (c.Ntotal + 1 > (1 << 17)) return fail(std::string(fn) + ": needs Ntotal + 1 <= 131072 (the fused update)");
  return 0;
}

extern "C" int dial_plan_set_instance_schedule(dial_plan* p, int b, float temp, int n_rows, const float* noise, void* stream) {
  static const char* fn = "dial_plan_set_instance_schedule";
  if (!p) return fail(std::string(fn) + ": null plan");
  if (int rc = need_instance(p, fn, b)) return rc;
  if (int rc = need_schedulable(p, fn)) return rc;
  const int n1 = p->hP.c.Hnode + 1;
  if (noise) {   // (the comparisons also reject NaN)
    if (!(temp > 0.f && temp <= FLT_MAX)) return fail(std::string(fn) + ": temp must be finite and > 0, got " + fmt_g(temp));
    if (n_rows < 1 || n_rows > DIAL_MAXDIFFUSE)
      return fail(std::string(fn) + ": n_rows " + std::to_string(n_rows) + " out of range (1.." DIAL_STR(DIAL_MAXDIFFUSE) ")");
    for (int i = 0; i < n_rows * n1; ++i)
      if (!(fabsf(noise[i]) <= FLT_MAX))
        return fail(std::string(fn) + ": noise[" + std::to_string(i / n1) + "][" + std::to_string(i % n1) + "] is not finite, got " + fmt_g(noise[i]));
  } else if (!p->sched.d) {
    return 0;   // no instance has a schedule: b already plans with the plan's own
  }
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  if (!p->sched.d && (e = p->sched.allocate(p->n_inst, 1, InstSchedule{})) != cudaSuccess)
    return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  e = p->sched.put(b, [&](InstSchedule* S) {
    memset(S, 0, sizeof(*S));
    if (!noise) return;
    S->on = 1; S->temp = temp; S->n_rows = n_rows;
    for (int r = 0; r < n_rows; ++r)
      for (int k = 0; k < n1; ++k) S->noise[r][k] = noise[r * n1 + k];
  }, st);
  p->key = launch_key(p);
  if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  return 0;
}

extern "C" int dial_plan_set_instance_iterations(dial_plan* p, const int32_t* n_iter, void* stream) {
  static const char* fn = "dial_plan_set_instance_iterations";
  if (!p || !n_iter) return fail(std::string(fn) + ": null argument");
  if (int rc = need_schedulable(p, fn)) return rc;
  for (int b = 0; b < p->n_inst; ++b)
    if (n_iter[b] < 0 || n_iter[b] > DIAL_MAXDIFFUSE)
      return fail(std::string(fn) + ": n_iter[" + std::to_string(b) + "] = " + std::to_string(n_iter[b]) + " out of range (0.." DIAL_STR(DIAL_MAXDIFFUSE) ")");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  if (!p->lims.d) {
    // first call: the rollout launches need instance-aligned CTAs from now on, the layout of per-instance
    // (or member) models, so those slots are allocated too, each holding the plan's model until one is set
    Staged<DevModel>& M = p->n_ens > 0 ? p->members : p->models;
    if (!M.d) e = M.allocate((size_t)p->n_inst * (p->n_ens > 0 ? p->n_ens : 1), 1, p->hM);
    if (e == cudaSuccess) e = p->lims.allocate(1, p->n_inst, DIAL_MAXDIFFUSE);
    if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  }
  e = p->lims.put(0, [&](int32_t* L) { memcpy(L, n_iter, sizeof(int32_t) * p->n_inst); }, st);
  p->key = launch_key(p);
  if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  return 0;
}

// The planning state (qpos, qvel, warm start, counters) and, on an ensemble plan, the planning models (member
// (b, 0) of each instance as the member slots hold it, else the plan's model), allocated by the first
// dial_plan_set_instance_delay or dial_plan_set_instance_observation; on failure the caller frees what it owns.
static cudaError_t allocate_planning(dial_plan* p, cudaStream_t st) {
  dial_plan::PlanningState& P = p->planning;
  if (P.qpos) return cudaSuccess;
  const size_t B = (size_t)p->n_inst, nq = p->hM.m.nq, nv = p->hM.m.nv;
  cudaError_t e = cudaSuccess;
  p->own(e, P.qpos, B * nq * sizeof(float), true, st);
  p->own(e, P.qvel, B * nv * sizeof(float), true, st);
  p->own(e, P.warm, B * nv * sizeof(float), true, st);
  p->own(e, P.cnt, B * 2 * sizeof(int32_t), true, st);
  if (p->n_ens > 0) p->own(e, P.models, B * sizeof(DevModel));
  for (size_t b = 0; P.models && b < B && e == cudaSuccess; ++b)
    e = p->members.d ? cudaMemcpyAsync(P.models + b, p->members.d + b * p->n_ens, sizeof(DevModel), cudaMemcpyDeviceToDevice, st)
                     : cudaMemcpy(P.models + b, &p->hM, sizeof(DevModel), cudaMemcpyHostToDevice);
  return e;
}

// First dial_plan_set_instance_delay: the settings and queues (and the planning state, if not yet allocated).
static cudaError_t allocate_delay(dial_plan* p, cudaStream_t st) {
  const size_t B = (size_t)p->n_inst, nu = p->hM.m.nu, mark = p->owned.size();
  dial_plan::DelayQueue& Q = p->queue;
  cudaError_t e = allocate_planning(p, st);
  if (e == cudaSuccess) e = p->delay.allocate(B, 1, DelaySetting{0, 0});
  p->own(e, Q.head, B * sizeof(int32_t), true, st);
  p->own(e, Q.ring, B * DIAL_MAXDELAY * nu * sizeof(float), true, st);
  p->own(e, Q.applied, B * nu * sizeof(float), true, st);
  p->own(e, Q.pending, B * DIAL_MAXDELAY * nu * sizeof(float), true, st);
  p->own(e, Q.len, B * sizeof(int32_t), true, st);
  if (e != cudaSuccess) { p->delay.release(); p->free_since(mark); }
  return e;
}

// First dial_plan_set_instance_observation: the settings, rings and observations (and the planning state, if
// not yet allocated).  Every ring starts empty.
static cudaError_t allocate_observation(dial_plan* p, cudaStream_t st) {
  const size_t B = (size_t)p->n_inst, nq = p->hM.m.nq, nv = p->hM.m.nv, nu = p->hM.m.nu, R = DIAL_OBSRING;
  const size_t mark = p->owned.size();
  cudaError_t e = allocate_planning(p, st);
  ObsSetting off;
  memset(&off, 0, sizeof(off));
  if (e == cudaSuccess) e = p->obs.allocate(B, 1, off);
  ObsBuffers& O = p->ob;
  p->own(e, O.ring, B * sizeof(ObsRing), true, st);
  p->own(e, O.rq, B * R * nq * sizeof(float), true, st);
  p->own(e, O.rv, B * R * nv * sizeof(float), true, st);
  p->own(e, O.rw, B * R * nv * sizeof(float), true, st);
  p->own(e, O.ra, B * R * nu * sizeof(float), true, st);
  p->own(e, O.rc, B * R * 2 * sizeof(int32_t), true, st);
  p->own(e, O.oq, B * nq * sizeof(float), true, st);
  p->own(e, O.ov, B * nv * sizeof(float), true, st);
  p->own(e, O.ow, B * nv * sizeof(float), true, st);
  p->own(e, O.oc, B * 2 * sizeof(int32_t), true, st);
  p->own(e, O.age, B * sizeof(int32_t), true, st);
  p->own(e, O.seq, B * DIAL_MAXDELAY * nu * sizeof(float), true, st);
  p->own(e, O.len, B * sizeof(int32_t), true, st);
  if (e != cudaSuccess) { p->obs.release(); p->free_since(mark); }
  return e;
}

extern "C" int dial_plan_set_instance_delay(dial_plan* p, int b, int steps, int predict, void* stream) {
  static const char* fn = "dial_plan_set_instance_delay";
  if (!p) return fail(std::string(fn) + ": null plan");
  if (int rc = need_instance(p, fn, b)) return rc;
  const dial_plan_desc& c = p->hP.c;
  if (c.Ntotal != c.Nsample || p->xch.on) return fail(std::string(fn) + ": sharded plans (Ntotal != Nsample) have no per-instance delay");
  if (steps < 0 || steps > DIAL_MAXDELAY)
    return fail(std::string(fn) + ": steps " + std::to_string(steps) + " out of range (0.." DIAL_STR(DIAL_MAXDELAY) ")");
  if (predict != 0 && predict != 1) return fail(std::string(fn) + ": predict must be 0 or 1, got " + std::to_string(predict));
  if (p->obs.d && steps + p->obs.h[b].k > DIAL_MAXDELAY)
    return fail(std::string(fn) + ": steps " + std::to_string(steps) + " plus instance " + std::to_string(b) +
                "'s observation delay " + std::to_string(p->obs.h[b].k) + " exceeds " DIAL_STR(DIAL_MAXDELAY));
  if (!p->mpc_bound) return fail(std::string(fn) + ": call dial_mpc_bind first (the queue is filled from the bound Y)");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  if (!p->delay.d && (e = allocate_delay(p, st)) != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  e = p->delay.put(b, [&](DelaySetting* s) { s->d = steps; s->predict = predict; }, st);
  p->key = launch_key(p);
  if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  const int n1 = c.Hnode + 1, nu = p->hM.m.nu;
  delay_refill_kernel<<<1, 128, 0, st>>>(b, steps, p->queue.head, p->queue.ring, p->mpc.Y, n1, nu, p->queue.pending);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int dial_plan_set_instance_observation(dial_plan* p, int b, int delay, const float* qpos_std,
                                                  const float* qvel_std, const uint32_t key[2], void* stream) {
  static const char* fn = "dial_plan_set_instance_observation";
  if (!p) return fail(std::string(fn) + ": null plan");
  if (int rc = need_instance(p, fn, b)) return rc;
  if (delay < 0 || delay > DIAL_MAXDELAY)
    return fail(std::string(fn) + ": delay " + std::to_string(delay) + " out of range (0.." DIAL_STR(DIAL_MAXDELAY) ")");
  const int d = p->delay.d ? p->delay.h[b].d : 0;
  if (delay + d > DIAL_MAXDELAY)
    return fail(std::string(fn) + ": delay " + std::to_string(delay) + " plus instance " + std::to_string(b) +
                "'s action delay " + std::to_string(d) + " exceeds " DIAL_STR(DIAL_MAXDELAY));
  const int nv = p->hM.m.nv;
  bool noisy = false;
  for (int w = 0; w < 2; ++w) {
    const float* sd = w == 0 ? qpos_std : qvel_std;
    for (int i = 0; sd && i < nv; ++i) {
      if (!(sd[i] >= 0.f) || !std::isfinite(sd[i]))
        return fail(std::string(fn) + ": " + (w == 0 ? "qpos_std[" : "qvel_std[") + std::to_string(i) + "] = " +
                    std::to_string(sd[i]) + " must be finite and >= 0");
      noisy |= sd[i] != 0.f;
    }
  }
  const dial_plan_desc& c = p->hP.c;
  if (c.Ntotal != c.Nsample || p->xch.on) return fail(std::string(fn) + ": sharded plans (Ntotal != Nsample) have no per-instance observation");
  if (!p->mpc_bound) return fail(std::string(fn) + ": call dial_mpc_bind first");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  if (!p->obs.d && (e = allocate_observation(p, st)) != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  e = p->obs.put(b, [&](ObsSetting* s) {
    s->k = delay; s->on = delay > 0 || noisy;
    s->key[0] = key ? key[0] : 0u; s->key[1] = key ? key[1] : 0u;
    for (int i = 0; i < 2 * DIAL_MAXV; ++i) s->sigma[i] = 0.f;
    for (int i = 0; i < nv; ++i) { s->sigma[i] = qpos_std ? qpos_std[i] : 0.f; s->sigma[nv + i] = qvel_std ? qvel_std[i] : 0.f; }
  }, st);
  p->key = launch_key(p);
  if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  observe_reset_kernel<<<1, 1, 0, st>>>(b, p->obs.d, p->ob.ring);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int dial_plan_set_instance_pushes(dial_plan* p, int b, int n, const dial_push* pushes, void* stream) {
  static const char* fn = "dial_plan_set_instance_pushes";
  if (!p) return fail(std::string(fn) + ": null plan");
  if (int rc = need_instance(p, fn, b)) return rc;
  if (n < 0 || n > DIAL_MAXPUSH)
    return fail(std::string(fn) + ": n " + std::to_string(n) + " out of range (0.." DIAL_STR(DIAL_MAXPUSH) ")");
  if (n > 0 && !pushes) return fail(std::string(fn) + ": null pushes");
  const int nbody = p->hM.m.nbody;
  for (int i = 0; i < n; ++i) {
    const dial_push& e = pushes[i];
    const std::string at = std::string(fn) + ": pushes[" + std::to_string(i) + "].";
    if (e.body < 1 || e.body >= nbody)
      return fail(at + "body " + std::to_string(e.body) + (e.body == 0 ? " is the world" : " out of range") +
                  " (1.." + std::to_string(nbody - 1) + ")");
    if (e.step < 1) return fail(at + "step must be >= 1, got " + std::to_string(e.step));
    if (e.n_steps < 1) return fail(at + "n_steps must be >= 1, got " + std::to_string(e.n_steps));
    for (int k = 0; k < 9; ++k) {
      const float x = k < 3 ? e.pos[k] : k < 6 ? e.force[k - 3] : e.torque[k - 6];
      if (!std::isfinite(x))
        return fail(at + (k < 3 ? "pos[" : k < 6 ? "force[" : "torque[") + std::to_string(k % 3) + "] is not finite, got " + fmt_g(x));
    }
  }
  const dial_plan_desc& c = p->hP.c;
  if (c.Ntotal != c.Nsample || p->xch.on) return fail(std::string(fn) + ": sharded plans (Ntotal != Nsample) have no per-instance pushes");
  if (!p->mpc_bound) return fail(std::string(fn) + ": call dial_mpc_bind first");
  if (n == 0 && !p->pushes.d) return 0;   // no instance has a table: b is already unpushed
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  if (!p->pushes.d) {
    PushTable none;
    memset(&none, 0, sizeof(none));
    if ((e = p->pushes.allocate(p->n_inst, 1, none)) != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  }
  e = p->pushes.put(b, [&](PushTable* T) {
    memset(T, 0, sizeof(*T));
    T->n = n;
    for (int i = 0; i < n; ++i) T->e[i] = pushes[i];
  }, st);
  p->key = launch_key(p);
  if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  return 0;
}

extern "C" int dial_plan_set_instance_plant(dial_plan* p, int b, const dial_plant* f, void* stream) {
  static const char* fn = "dial_plan_set_instance_plant";
  if (!p) return fail(std::string(fn) + ": null plan");
  if (int rc = need_instance(p, fn, b)) return rc;
  if (f) {   // (the comparisons also reject NaN)
    const std::string at = std::string(fn) + ": ";
    if (f->substeps < 1 || f->substeps > DIAL_MAXSUBSTEPS)
      return fail(at + "substeps " + std::to_string(f->substeps) + " out of range (1.." DIAL_STR(DIAL_MAXSUBSTEPS) ")");
    if (f->iterations < 1 || f->iterations > 100)
      return fail(at + "iterations " + std::to_string(f->iterations) + " out of range (1..100)");
    if (f->ls_iterations < 1 || f->ls_iterations > 50)
      return fail(at + "ls_iterations " + std::to_string(f->ls_iterations) + " out of range (1..50)");
    if (!(f->tolerance >= 0.f && f->tolerance <= FLT_MAX))
      return fail(at + "tolerance must be finite and >= 0, got " + fmt_g(f->tolerance));
  }
  const dial_plan_desc& c = p->hP.c;
  if (c.Ntotal != c.Nsample || p->xch.on) return fail(std::string(fn) + ": sharded plans (Ntotal != Nsample) have no per-instance plant");
  if (!p->mpc_bound) return fail(std::string(fn) + ": call dial_mpc_bind first");
  if (!f && !p->plant_models.d) return 0;   // no instance has a setting: b already steps like its planner
  cudaStream_t st = (cudaStream_t)stream;
  const size_t B = (size_t)p->n_inst;
  cudaError_t e = cudaSuccess;
  if (!p->plant_models.d) {
    // first setting: every plant slot holds its instance's model (uploaded synchronously: nothing reads the
    // slots yet), every plan slot the plan's descriptor, every instance is in the group of substeps 1
    p->plant.assign(B, dial_plant{0, 0, 0, 0.f});
    if ((e = p->plant_models.allocate(B, 1, p->hM)) == cudaSuccess && p->models.d) {
      for (size_t i = 0; i < B; ++i) p->plant_models.h[i] = p->models.h[i];
      e = cudaMemcpy(p->plant_models.d, p->plant_models.h, B * sizeof(DevModel), cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess) e = p->plant_plans.allocate(DIAL_MAXSUBSTEPS, 1, p->hP);
    if (e == cudaSuccess && B > 1) e = p->plant_mask.allocate(DIAL_MAXSUBSTEPS, B, 0);
    if (e == cudaSuccess && B > 1) e = p->plant_mask.put(0, [&](int32_t* M) { for (size_t i = 0; i < B; ++i) M[i] = 1; }, st);
    if (e != cudaSuccess) {
      p->plant_models.release(); p->plant_plans.release(); p->plant_mask.release(); p->plant.clear();
      return fail(std::string(fn) + ": " + cudaGetErrorString(e));
    }
  }
  const int k0 = plant_substeps(p, b);
  p->plant[b] = f ? *f : dial_plant{0, 0, 0, 0.f};
  const int k1 = plant_substeps(p, b);
  const uint32_t ks0 = p->key.plant_ks;
  p->key = launch_key(p);
  e = p->plant_models.put(b, [&](DevModel* h) { *h = plant_model(p, b); }, st);
  // the groups b left and joined; the plan slots of substep counts that came into use
  for (int k : {k0, k1})
    if (e == cudaSuccess && B > 1 && k0 != k1)
      e = p->plant_mask.put(k - 1, [&](int32_t* M) { for (size_t i = 0; i < B; ++i) M[i] = plant_substeps(p, (int)i) == k; }, st);
  if (e == cudaSuccess) e = put_plant_plans(p, p->key.plant_ks & ~ks0, st);
  if (e != cudaSuccess) return fail(std::string(fn) + ": " + cudaGetErrorString(e));
  return 0;
}

extern "C" int dial_plan_set_instance_terrain(dial_plan* p, int b, int side, const dial_terrain* t, void* stream) {
  static const char* fn = "dial_plan_set_instance_terrain";
  if (!p) return fail(std::string(fn) + ": null plan");
  if (int rc = need_instance(p, fn, b)) return rc;
  const std::string at = std::string(fn) + ": ";
  if (side != DIAL_TERRAIN_PLANT && side != DIAL_TERRAIN_PLANNER)
    return fail(at + "side " + std::to_string(side) + " out of range (0 plant, 1 planner)");
  if (t) {
    if (t->nx < 2 || t->nx > DIAL_MAXTERRAIN || t->ny < 2 || t->ny > DIAL_MAXTERRAIN)
      return fail(at + "grid " + std::to_string(t->nx) + " x " + std::to_string(t->ny) + " out of range (2.." DIAL_STR(DIAL_MAXTERRAIN) " per side)");
    if (!(t->spacing > 0.f && t->spacing <= FLT_MAX)) return fail(at + "spacing must be finite and > 0, got " + fmt_g(t->spacing));
    if (!std::isfinite(t->x0) || !std::isfinite(t->y0)) return fail(at + "origin must be finite, got (" + fmt_g(t->x0) + ", " + fmt_g(t->y0) + ")");
    if (!t->heights) return fail(at + "null heights");
    for (int j = 0; j < t->ny; ++j)
      for (int i = 0; i < t->nx; ++i)
        if (!std::isfinite(t->heights[(size_t)j * t->nx + i]))
          return fail(at + "heights[" + std::to_string(j) + "][" + std::to_string(i) + "] is not finite, got " + fmt_g(t->heights[(size_t)j * t->nx + i]));
  }
  const dial_model_desc& m = p->hM.m;
  bool floor = false;
  for (int k = 0; k < m.npair; ++k)
    floor |= (m.pair_kind[k] == PAIR_PLANE_SPHERE || m.pair_kind[k] == PAIR_PLANE_CAPSULE) && m.geom_bodyid[m.pair_geom1[k]] == 0;
  if (!floor) return fail(at + "the model has no floor pair (a plane geom on the world body against a sphere or capsule)");
  if (p->hM.dense) return fail(at + "the dense solver path has no terrain build");
  if (!p->kernels.terrain) return fail(at + "this custom build has no terrain kernel (compile it with DIAL_TERRAIN)");
  const dial_plan_desc& c = p->hP.c;
  if (c.Ntotal != c.Nsample || p->xch.on) return fail(at + "sharded plans (Ntotal != Nsample) have no per-instance terrain");
  if (!p->mpc_bound) return fail(at + "call dial_mpc_bind first");
  Staged<DevTerrain>& D = p->terrain[side];
  if (!t && !D.d) return 0;   // no instance has a terrain on this side: b is already flat
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  if (!D.d) {   // first terrain on this side: flat descriptors, no heights yet
    DevTerrain flat;
    memset(&flat, 0, sizeof(flat));
    if ((e = D.allocate(p->n_inst, 1, flat)) != cudaSuccess) return fail(at + cudaGetErrorString(e));
    p->heights[side].assign(p->n_inst, Staged<float>());
  }
  Staged<float>& Hs = p->heights[side][b];
  const size_t n = t ? (size_t)t->nx * t->ny : 0;
  if (t && (!Hs.d || Hs.width < n)) {
    // a table larger than b's allocation: a new one (the old one is freed once the device is idle), and the
    // graphs are captured again
    Staged<float> grown;
    if ((e = grown.allocate(1, n, 0.f)) != cudaSuccess) return fail(at + cudaGetErrorString(e));
    if ((e = cudaDeviceSynchronize()) != cudaSuccess) { grown.release(); return fail(at + cudaGetErrorString(e)); }
    Hs.release();
    Hs = grown;
    drop_graphs(p);
  }
  if (t) e = Hs.put(0, [&](float* h) { memcpy(h, t->heights, n * sizeof(float)); }, st);
  if (e == cudaSuccess)
    e = D.put(b, [&](DevTerrain* T) {
      memset(T, 0, sizeof(*T));
      if (!t) return;
      T->nx = t->nx; T->ny = t->ny; T->x0 = t->x0; T->y0 = t->y0; T->inv = 1.f / t->spacing; T->h = Hs.d;
    }, st);
  p->key = launch_key(p);
  if (e != cudaSuccess) return fail(at + cudaGetErrorString(e));
  return 0;
}

extern "C" int dial_plan_observed_state(dial_plan* p, float* qpos, float* qvel, float* warm, int32_t* counters,
                                        int32_t* age, void* stream) {
  static const char* fn = "dial_plan_observed_state";
  if (!p) return fail(std::string(fn) + ": null plan");
  if (!p->mpc_bound) return fail(std::string(fn) + ": call dial_mpc_bind first");
  const size_t B = (size_t)p->n_inst, nq = p->hM.m.nq, nv = p->hM.m.nv;
  // the observation of the last step when it ran the observe launch, else the plant state at age 0
  const bool ob = p->ran.obs;
  cudaStream_t st = (cudaStream_t)stream;
  const auto cp = [&](void* dst, const void* src, size_t bytes) {
    return dst ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st) : cudaSuccess;
  };
  CUDA_OK(cp(qpos, ob ? p->ob.oq : p->mpc.qpos, B * nq * sizeof(float)));
  CUDA_OK(cp(qvel, ob ? p->ob.ov : p->mpc.qvel, B * nv * sizeof(float)));
  CUDA_OK(cp(warm, ob ? p->ob.ow : p->mpc.qacc_warmstart, B * nv * sizeof(float)));
  CUDA_OK(cp(counters, ob ? p->ob.oc : p->mpc.counters, B * 2 * sizeof(int32_t)));
  if (age) {
    if (ob) CUDA_OK(cp(age, p->ob.age, B * sizeof(int32_t)));
    else CUDA_OK(cudaMemsetAsync(age, 0, B * sizeof(int32_t), st));
  }
  return 0;
}

extern "C" int dial_plan_pending_actions(dial_plan* p, float* out, void* stream) {
  static const char* fn = "dial_plan_pending_actions";
  if (!p || !out) return fail(std::string(fn) + ": null argument");
  const size_t n = (size_t)p->n_inst * DIAL_MAXDELAY * p->hM.m.nu * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  if (p->queue.pending) CUDA_OK(cudaMemcpyAsync(out, p->queue.pending, n, cudaMemcpyDeviceToDevice, st));
  else CUDA_OK(cudaMemsetAsync(out, 0, n, st));
  return 0;
}

extern "C" int dial_plan_planning_state(dial_plan* p, float* qpos, float* qvel, float* warm, int32_t* counters, void* stream) {
  static const char* fn = "dial_plan_planning_state";
  if (!p) return fail(std::string(fn) + ": null plan");
  if (!p->mpc_bound) return fail(std::string(fn) + ": call dial_mpc_bind first");
  const size_t B = (size_t)p->n_inst, nq = p->hM.m.nq, nv = p->hM.m.nv;
  // the last step planned from the planning state when it predicted or observed (then the other instances'
  // rows hold their plant state, copied in that step)
  const bool pred = p->ran.planning();
  cudaStream_t st = (cudaStream_t)stream;
  const auto cp = [&](void* dst, const void* src, size_t bytes) {
    return dst ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st) : cudaSuccess;
  };
  const dial_plan::PlanningState& P = p->planning;
  CUDA_OK(cp(qpos, pred ? P.qpos : p->mpc.qpos, B * nq * sizeof(float)));
  CUDA_OK(cp(qvel, pred ? P.qvel : p->mpc.qvel, B * nv * sizeof(float)));
  CUDA_OK(cp(warm, pred ? P.warm : p->mpc.qacc_warmstart, B * nv * sizeof(float)));
  CUDA_OK(cp(counters, pred ? P.cnt : p->mpc.counters, B * 2 * sizeof(int32_t)));
  return 0;
}

extern "C" int dial_plan_get_task(const dial_plan* p, dial_task* out) {
  if (!p || !out) return fail("dial_plan_get_task: null argument");
  const dial_task& t = plan_task(p->hP.c);   // the plan's task block (include/dial_b200.h)
  if (!task_valid(t)) return fail("dial_plan_get_task: the plan's n_stage / n_user are out of range (1..DIAL_MAXSTAGE / 0..DIAL_MAXUSER)");
  *out = t;
  return 0;
}

extern "C" int dial_env_step(dial_plan* p, const dial_state* s, const float* action, float* qpos_out,
                             float* qvel_out, float* warm_out, float* reward, float* ctrl_out, void* stream) {
  return dial_env_step_kin(p, s, action, qpos_out, qvel_out, warm_out, reward, ctrl_out, nullptr, stream);
}

extern "C" int dial_env_step_kin(dial_plan* p, const dial_state* s, const float* action, float* qpos_out,
                                 float* qvel_out, float* warm_out, float* reward, float* ctrl_out, float* kin_out,
                                 void* stream) {
  if (!p || !s || !action || !qpos_out || !qvel_out || !warm_out || !reward) return fail("dial_env_step: null argument");
  RolloutArgs A; memset(&A, 0, sizeof(A));
  fill_state(A, s);
  A.nrows = 1; A.H = 1; A.mode = 0; A.us = action; A.rewss = reward;
  A.qpos_out = qpos_out; A.qvel_out = qvel_out; A.warm_out = warm_out; A.ctrl_out = ctrl_out; A.kin_out = kin_out;
  CUDA_OK(launch_rollout(p, A, 1, (cudaStream_t)stream));
  return 0;
}

extern "C" int dial_pipeline_init(dial_plan* p, const float* qpos, const float* qvel, float* qpos_out,
                                  float* warm_out, void* stream) {
  if (!p || !qpos || !qvel || !qpos_out || !warm_out) return fail("dial_pipeline_init: null argument");
  RolloutArgs A; memset(&A, 0, sizeof(A));
  A.qpos0 = qpos; A.qvel0 = qvel; A.warm0 = p->zeros;  // mjx.make_data: qacc_warmstart = 0
  A.nrows = 1; A.H = 1; A.mode = 2; A.qpos_out = qpos_out; A.warm_out = warm_out;
  CUDA_OK(launch_rollout(p, A, 1, (cudaStream_t)stream));
  return 0;
}

extern "C" int dial_reverse_rollout(dial_plan* p, const dial_state* s, const float* eps, const uint32_t key[2],
                                    const float* Ybar, const float* noise_scale, float* rews_local, void* stream) {
  if (!p || !s || !Ybar || !noise_scale || !rews_local) return fail("dial_reverse_rollout: null argument");
  if (p->n_inst > 1) return fail("dial_reverse_rollout: batched plans run through dial_mpc_step");
  if (!eps && !key) return fail("dial_reverse_rollout: need eps or key");
  RolloutArgs A; memset(&A, 0, sizeof(A));
  fill_state(A, s);
  const dial_plan_desc& c = p->hP.c;
  A.nrows = c.Nsample + 1; A.H = c.Hsample + 1; A.mode = 1;
  A.eps = eps; A.Ybar = Ybar; A.noise = noise_scale;
  if (key) { A.key0 = key[0]; A.key1 = key[1]; }
  p->cur ^= 1;
  A.rews = rews_local; A.q = p->traj_q[p->cur]; A.qd = p->traj_qd[p->cur]; A.xpos = p->traj_x[p->cur];
  A.dbg = p->dbg;
  fill_xch(p, A);   // sharded plans with a connected exchange: rewards go straight to every rank's mailbox
  CUDA_OK(launch_rollout_any(p, A, (cudaStream_t)stream));
  return 0;
}

extern "C" int dial_reverse_update(dial_plan* p, const float* eps, const uint32_t key[2], const float* Ybar,
                                   const float* noise_scale, const float* rews_all, float* Ybar_out,
                                   float* weights, void* stream) {
  return dial_reverse_update_x(p, eps, key, Ybar, noise_scale, rews_all, Ybar_out, weights, nullptr, stream);
}

extern "C" int dial_reverse_update_x(dial_plan* p, const float* eps, const uint32_t key[2], const float* Ybar,
                                     const float* noise_scale, const float* rews_all, float* Ybar_out,
                                     float* weights, float* rews_gathered, void* stream) {
  if (!p || !Ybar || !noise_scale || !Ybar_out) return fail("dial_reverse_update: null argument");
  if (p->n_inst > 1) return fail("dial_reverse_update: batched plans run through dial_mpc_step");
  if (!rews_all && !p->xch.on) return fail("dial_reverse_update: rews_all may be NULL only with a connected exchange");
  if (!eps && !key) return fail("dial_reverse_update: need eps or key");
  const dial_plan_desc& c = p->hP.c;
  cudaStream_t st = (cudaStream_t)stream;
  float* w = weights ? weights : p->weights;
  // rews_all == NULL: the rewards are in this rank's mailbox (written by every rank's rollout
  // epilogue over NVLink); the kernel waits for the flags, and rews_gathered gets a compact copy
  XchWait X = xch_wait_args(p, rews_gathered);
  if (rews_all) X.mbox = nullptr;
  weights_kernel<<<1, 1024, 0, st>>>(rews_all, c.Ntotal + 1, c.temp_sample, w, X);
  p->launches++;
  CUDA_OK(cudaGetLastError());
  ybar_kernel<<<p->ybar_grid, YBAR_THREADS, 0, st>>>(w, eps, key ? key[0] : 0u, key ? key[1] : 0u, Ybar, noise_scale,
                                                     c.Ntotal, c.Hnode + 1, p->hM.m.nu, p->partial, p->counter, Ybar_out, nullptr);
  p->launches++;
  CUDA_OK(cudaGetLastError());
  if (weights && weights != p->weights)
    CUDA_OK(cudaMemcpyAsync(p->weights, weights, ((size_t)c.Ntotal + 1) * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// The fused update of every instance of the plan: the one launch of update_kernel, used by the
// control-step graph (mpc_enqueue) and by dial_reverse_update_fused.  Grid upd_grid x n_inst over the
// plan's partials and per-instance counters.  The control-step graph passes the schedules, the limits, the
// iteration `iter` and the previous iteration's weights buffer `weights_prev` (what a skipped instance
// forwards); dial_reverse_update_fused passes none.
static int launch_update(dial_plan* p, const float* rews, float* weights, const XchWait& X, uint32_t* rng,
                         const float* Ybar, const float* noise, float* Ybar_out, cudaStream_t st,
                         const InstSchedule* sched = nullptr, const int32_t* iter_lim = nullptr, int iter = 0,
                         const float* weights_prev = nullptr) {
  const dial_plan_desc& c = p->hP.c;
  update_kernel<<<dim3(p->upd_grid, p->n_inst), YBAR_THREADS, 0, st>>>(rews, c.Ntotal + 1, c.temp_sample, weights, X, rng, Ybar,
                                                                     noise, c.Ntotal, c.Hnode + 1, p->hM.m.nu, p->partial,
                                                                     p->counter, Ybar_out, sched, iter_lim, iter,
                                                                     weights_prev ? weights_prev : weights);
  p->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int dial_reverse_update_fused(dial_plan* p, const float* rews, uint32_t* rng, const float* Ybar,
                                         const float* noise_scale, float* Ybar_out, float* weights, void* stream) {
  if (!p || !rews || !rng || !Ybar || !noise_scale || !Ybar_out || !weights) return fail("dial_reverse_update_fused: null argument");
  const dial_plan_desc& c = p->hP.c;
  if (c.Ntotal != c.Nsample) return fail("dial_reverse_update_fused: sharded plans (Ntotal != Nsample) are not supported");
  if (c.Ntotal + 1 > (1 << 17)) return fail("dial_reverse_update_fused: needs Ntotal + 1 <= 131072 (the fused update)");
  XchWait X; memset(&X, 0, sizeof(X));
  return launch_update(p, rews, weights, X, rng, Ybar, noise_scale, Ybar_out, (cudaStream_t)stream);
}

// the bars of every instance of the plan (the control-step graph; the public call below is single-instance);
// with iteration limits (iter_lim, iteration `iter`) the instance-indexed kernels run, also for one instance
static int enqueue_trajbar(dial_plan* p, const float* weights, int rank, float* qbar, float* qdbar, float* xbar,
                           cudaStream_t st, const int32_t* iter_lim = nullptr, int iter = 0) {
  const dial_plan_desc& c = p->hP.c;
  const dial_model_desc& m = p->hM.m;
  const float* w = weights ? weights : p->weights;
  const int H = c.Hsample + 1, rows = c.Nsample + 1;
  TrajArgs T;
  T.traj[0] = p->traj_q[p->cur]; T.traj[1] = p->traj_qd[p->cur]; T.traj[2] = p->traj_x[p->cur];
  T.out[0] = qbar; T.out[1] = qdbar; T.out[2] = xbar;
  const bool xsum = p->xch.on && qbar && qdbar && xbar;   // sum over ranks on the device (peer memory)
  if (xsum) {
    T.out[0] = p->xch.bars_partial; T.out[1] = T.out[0] + (size_t)H * m.nq; T.out[2] = T.out[1] + (size_t)H * m.nv;
  }
  T.ncol[0] = m.nq; T.ncol[1] = m.nv; T.ncol[2] = 3 * (m.nbody - 1);
  T.coloff[0] = 0; T.coloff[1] = m.nq; T.coloff[2] = m.nq + m.nv;
  T.coltot = m.nq + m.nv + 3 * (m.nbody - 1);
  T.nrows = rows; T.inst_rows = (p->n_ens > 1 ? p->n_ens : 1) * rows; T.H = H; T.weights = w; T.w_offset = c.shard_offset; T.mean_row = c.Nsample;
  T.mean_weight_index = c.Ntotal; T.include_mean = rank == 0 ? 1 : 0; T.partial = p->tb_partial;
  const int maxlen = H * (T.ncol[2] > T.ncol[0] ? T.ncol[2] : T.ncol[0]);   // nq = nv + 1 > nv always
  const dim3 g1((maxlen + 255) / 256, TB_CHUNKS, 3 * p->n_inst), g2(H, p->n_inst);
  const bool batch = p->n_inst > 1 || iter_lim;
  if (batch) trajbar_partial_kernel<true><<<g1, 256, 0, st>>>(T, iter_lim, iter);
  else trajbar_partial_kernel<false><<<g1, 256, 0, st>>>(T, nullptr, 0);
  p->launches++;
  CUDA_OK(cudaGetLastError());
  if (batch) trajbar_final_kernel<true><<<g2, 128, 0, st>>>(T, iter_lim, iter);
  else trajbar_final_kernel<false><<<g2, 128, 0, st>>>(T, nullptr, 0);
  p->launches++;
  CUDA_OK(cudaGetLastError());
  if (xsum) {
    BarsXch Bx; memset(&Bx, 0, sizeof(Bx));
    for (int r = 0; r < p->xch.world; ++r) { Bx.mbox[r] = p->xch.bars(r); Bx.flags[r] = p->xch.bflags(r); }
    Bx.seq = p->xch.bseq(); Bx.err = p->xch.err(); Bx.world = p->xch.world; Bx.rank = p->xch.rank; Bx.nbar = p->xch.nbar;
    Bx.partial = p->xch.bars_partial; Bx.out[0] = qbar; Bx.out[1] = qdbar; Bx.out[2] = xbar;
    Bx.n0 = H * m.nq; Bx.n1 = H * m.nv;
    bars_allreduce_kernel<<<1, 1024, 0, st>>>(Bx);
    p->launches++;
    CUDA_OK(cudaGetLastError());
  }
  return 0;
}

extern "C" int dial_reverse_trajbar(dial_plan* p, const float* weights, int rank, float* qbar, float* qdbar,
                                    float* xbar, void* stream) {
  if (!p) return fail("dial_reverse_trajbar: null plan");
  if (p->n_inst > 1) return fail("dial_reverse_trajbar: batched plans run through dial_mpc_step");
  return enqueue_trajbar(p, weights, rank, qbar, qdbar, xbar, (cudaStream_t)stream);
}

// ---- multi-GPU exchange over NVLink peer memory -------------------------------------------------
extern "C" int dial_exchange_create(dial_plan* p, int rank, int world, unsigned char handle_out[DIAL_IPC_HANDLE_BYTES]) {
  if (!p || !handle_out) return fail("dial_exchange_create: null argument");
  if (world < 2 || world > DIAL_MAXRANK || rank < 0 || rank >= world) return fail("dial_exchange_create: need 2 <= world <= DIAL_MAXRANK");
  static_assert(sizeof(cudaIpcMemHandle_t) <= DIAL_IPC_HANDLE_BYTES, "IPC handle does not fit");
  const dial_plan_desc& c = p->hP.c;
  const dial_model_desc& m = p->hM.m;
  if (c.Ntotal != c.Nsample * world || c.shard_offset != rank * c.Nsample) return fail("dial_exchange_create: plan shard does not match rank/world");
  if (p->xch.base[p->xch.rank]) return fail("dial_exchange_create: already created");
  dial_plan::Exchange& x = p->xch;
  x.rank = rank; x.world = world;
  x.nbar = (c.Hsample + 1) * (m.nq + m.nv + 3 * (m.nbody - 1));
  auto up = [](size_t n) { return (n + 31) & ~(size_t)31; };
  size_t o = 0;
  x.o_mbox = o; o += up(2 * ((size_t)c.Ntotal + 1));
  x.o_bars = o; o += up(2 * (size_t)DIAL_MAXRANK * x.nbar);
  x.o_flags = o; o += up(2 * DIAL_MAXRANK);
  x.o_bflags = o; o += up(2 * DIAL_MAXRANK);
  x.o_local = o; o += 32;
  x.words = o;
  void* d = nullptr;
  CUDA_OK(cudaMalloc(&d, x.words * sizeof(uint32_t)));
  CUDA_OK(cudaMemset(d, 0, x.words * sizeof(uint32_t)));
  x.base[rank] = reinterpret_cast<uint32_t*>(d);
  CUDA_OK(cudaMalloc(&x.bars_partial, (size_t)x.nbar * sizeof(float)));
  cudaIpcMemHandle_t h;
  CUDA_OK(cudaIpcGetMemHandle(&h, d));
  memset(handle_out, 0, DIAL_IPC_HANDLE_BYTES);
  memcpy(handle_out, &h, sizeof(h));
  return 0;
}

extern "C" int dial_exchange_connect(dial_plan* p, const unsigned char* handles) {
  if (!p || !handles) return fail("dial_exchange_connect: null argument");
  dial_plan::Exchange& x = p->xch;
  if (!x.base[x.rank]) return fail("dial_exchange_connect: call dial_exchange_create first");
  for (int r = 0; r < x.world; ++r) {
    if (r == x.rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)r * DIAL_IPC_HANDLE_BYTES, sizeof(h));
    void* d = nullptr;
    CUDA_OK(cudaIpcOpenMemHandle(&d, h, cudaIpcMemLazyEnablePeerAccess));
    x.base[r] = reinterpret_cast<uint32_t*>(d);
  }
  x.on = true;
  return 0;
}

extern "C" int dial_exchange_status(dial_plan* p, uint32_t out[6]) {
  if (!p || !out) return fail("dial_exchange_status: null argument");
  if (!p->xch.on) { for (int i = 0; i < 6; ++i) out[i] = 0; return 0; }
  CUDA_OK(cudaMemcpy(out, p->xch.base[p->xch.rank] + p->xch.o_local, 6 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int dial_reverse_trajectories(dial_plan* p, float* q, float* qd, float* xpos, void* stream) {
  if (!p) return fail("dial_reverse_trajectories: null plan");
  if (p->n_inst > 1) return fail("dial_reverse_trajectories: batched plans run through dial_mpc_step");
  const dial_plan_desc& c = p->hP.c;
  const dial_model_desc& m = p->hM.m;
  const size_t n = ((size_t)c.Nsample + 1) * (c.Hsample + 1) * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  if (q) CUDA_OK(cudaMemcpyAsync(q, p->traj_q[p->cur], n * m.nq, cudaMemcpyDeviceToDevice, st));
  if (qd) CUDA_OK(cudaMemcpyAsync(qd, p->traj_qd[p->cur], n * m.nv, cudaMemcpyDeviceToDevice, st));
  if (xpos) CUDA_OK(cudaMemcpyAsync(xpos, p->traj_x[p->cur], n * 3 * (m.nbody - 1), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// ---- device-resident synchronous MPC loop ---------------------------------------------------
extern "C" int dial_mpc_bind(dial_plan* p, const dial_mpc_buffers* b, const float* M_shift) {
  if (!p || !b || !M_shift) return fail("dial_mpc_bind: null argument");
  if (!b->qpos || !b->qvel || !b->qacc_warmstart || !b->counters || !b->rng || !b->Y || !b->ctrl || !b->reward ||
      !b->rews || !b->noise)
    return fail("dial_mpc_bind: only qbar/qdbar/xbar may be null");
  const dial_plan_desc& c = p->hP.c;
  if (c.Ntotal != c.Nsample && !p->xch.on)
    return fail("dial_mpc_bind: a sharded plan needs a connected exchange (dial_exchange_create / dial_exchange_connect) for the device-resident loop");
  if (c.Ntotal != c.Nsample && !b->rews_all) return fail("dial_mpc_bind: sharded plans need rews_all [Ntotal+1]");
  if (p->n_inst > 1 && b->rews_all) return fail("dial_mpc_bind: rews_all must be NULL on a batched plan");
  const int n1 = c.Hnode + 1, nu = p->hM.m.nu;
  drop_graphs(p);
  cudaError_t e = cudaSuccess;
  if (!p->mpc_Msh) CUDA_OK(p->own(e, p->mpc_Msh, DIAL_MAXNODE * DIAL_MAXNODE * sizeof(float)));
  if (!p->mpc_Y1) CUDA_OK(p->own(e, p->mpc_Y1, (size_t)p->n_inst * DIAL_MAXNODE * DIAL_MAXU * sizeof(float)));
  if (!p->mpc_key) CUDA_OK(p->own(e, p->mpc_key, 2 * sizeof(uint32_t)));
  CUDA_OK(cudaMemcpy(p->mpc_Msh, M_shift, (size_t)n1 * n1 * sizeof(float), cudaMemcpyHostToDevice));
  (void)nu;
  p->mpc = *b;
  p->mpc_bound = true;
  return 0;
}

// enqueue one MPC step on `st` (eagerly or into a capture), the launch sequence of the plan's key `k`
static int mpc_enqueue(dial_plan* p, const LaunchKey& k, int n_diffuse, int env_step, cudaStream_t st) {
  const dial_plan_desc& c = p->hP.c;
  const dial_mpc_buffers& B = p->mpc;
  const int n1 = c.Hnode + 1, nu = p->hM.m.nu, ni = p->n_inst;
  const int K = p->n_ens > 1 ? p->n_ens : 1;   // rollout rows per sample
  const bool batched = ni > 1;
  const dial_plan::DelayQueue& Q = p->queue;
  const dial_plan::PlanningState& P = p->planning;
  // the terrain tables the plant's env step and the planner's launches read (null: every instance on the floor)
  const DevTerrain* plant_terrain = k.terrain[DIAL_TERRAIN_PLANT] ? p->terrain[DIAL_TERRAIN_PLANT].d : nullptr;
  const DevTerrain* planner_terrain = k.terrain[DIAL_TERRAIN_PLANNER] ? p->terrain[DIAL_TERRAIN_PLANNER].d : nullptr;
  float* Y[2] = {B.Y, p->mpc_Y1};
  int cur = 0;
  // control latency, once some instance was given a delay: the queues move in a step with an env step, which
  // then applies the action each queue pops (Q.applied, one row of nu per instance) instead of Y[b][0]; while
  // some instance predicts, the queue launch also lays out the pending actions in the other steps
  if (k.delay && (env_step == 1 || k.predicts)) {
    delay_queue_kernel<<<ni, 128, 0, st>>>(p->delay.d, Q.head, Q.ring, Y[cur], n1, nu, env_step == 1,
                                           Q.applied, Q.pending, Q.len);
    p->launches++;
    CUDA_OK(cudaGetLastError());
  }
  const float* act = k.delay ? Q.applied : Y[cur];
  const int act_n1 = k.delay ? 1 : n1;   // rows of nu floats between two instances' actions
  // ensemble adaptation, once some instance has turned it on: before the plant's env step, member (b, k)
  // makes the same env step on its own model, from instance b's state, counters and task with the action
  // the plant applies (row b K + k, its CTA staging member slot b K + k); only the post-step qvel is kept
  const bool adapt = env_step == 1 && k.adapt;
  if (adapt) {
    ens_gather_kernel<<<ni, 128, 0, st>>>(act, K, act_n1, nu, p->pred_us);
    p->launches++;
    CUDA_OK(cudaGetLastError());
    RolloutArgs A; memset(&A, 0, sizeof(A));
    A.qpos0 = B.qpos; A.qvel0 = B.qvel; A.warm0 = B.qacc_warmstart; A.counters_in = B.counters;
    A.nrows = ni * K; A.H = 1; A.mode = 0; A.us = p->pred_us;
    A.rows_per_inst = K; A.rows_per_model = 1; A.models = p->members.d;
    if (B.tasks) { A.tasks = B.tasks; A.task_rows = K; }
    A.qd = p->pred_qd;
    A.terrain = planner_terrain;
    CUDA_OK(launch_rollout(p, A, 1, st));
  }
  if (env_step == 1) {
    // state = step_env(state, Y0[0])  (dial_core.py:245): in place, counters advanced by the kernel;
    // batched: row b is instance b, its action Y[b][0]
    RolloutArgs A; memset(&A, 0, sizeof(A));
    A.qpos0 = B.qpos; A.qvel0 = B.qvel; A.warm0 = B.qacc_warmstart;
    A.counters_in = B.counters; A.counters_out = B.counters;
    A.nrows = ni; A.H = 1; A.mode = 0; A.us = act; A.rewss = B.reward;
    if (batched) { A.rows_per_inst = 1; A.us_row = act_n1 * nu; }
    if (B.tasks) { A.tasks = B.tasks; A.task_rows = batched ? 1 : 0; }
    A.models = p->models.d;
    A.qpos_out = B.qpos; A.qvel_out = B.qvel; A.warm_out = B.qacc_warmstart; A.ctrl_out = B.ctrl;
    A.terrain = plant_terrain;
    if (!k.plant) CUDA_OK(launch_rollout(p, A, 1, st));
    // with plant fidelities: one launch of the generic kernel per distinct substep count k, on the plant slots
    // and the plan descriptor of k; batched, the rows of the other groups exit at entry (mask k as the
    // launch's iteration limits, iteration 0), so every instance's state, counters, reward and ctrl are
    // written once
    for (int s_ = 0; k.plant && s_ < DIAL_MAXSUBSTEPS; ++s_) {
      if (!((k.plant_ks >> s_) & 1u)) continue;
      A.models = p->plant_models.d;
      if (batched) { A.iter_lim = p->plant_mask.d + (size_t)s_ * ni; A.iter = 0; }
      CUDA_OK(launch_rollout(p, A, 1, st, p->plant_plans.d + s_, true));
    }
  }
  if (adapt) {   // each adapting instance's belief from its members' predictions and the observed qvel
    ens_belief_kernel<<<ni, 32, 0, st>>>(p->pred_qd, B.qvel, p->adapt.d, K, p->hM.m.nv, p->belief_L.d, p->belief_w.d, p->dEll);
    p->launches++;
    CUDA_OK(cudaGetLastError());
  }
  if (env_step == 1 && k.push) {   // pushes, on the post-step plant state; dt: the env step's duration
    const double dt = (double)c.n_frames * (double)p->hM.m.timestep;
    push_kernel<<<ni, 32, 0, st>>>(p->dM, p->models.d, p->pushes.d, B.counters, B.qpos, B.qvel, dt);
    p->launches++;
    CUDA_OK(cudaGetLastError());
  }
  if (env_step == 1 || env_step == 2) {
    // Y0 = shift(Y0)  (dial_core.py:252)
    mpc_shift_kernel<<<ni, DIAL_MAXNODE * DIAL_MAXU, 0, st>>>(p->mpc_Msh, Y[cur], Y[cur ^ 1], n1, nu);
    p->launches++;
    CUDA_OK(cudaGetLastError());
    cur ^= 1;
  }
  // The planning state: the plant state, or once some instance predicts, a copy of it in which each predicting
  // instance b takes d_b env steps with its queued actions on its planning model (launch j: one row per
  // instance, action pending[b][j], in place; an instance with pred_len[b] <= j exits at entry)
  // With the observe launch (once some instance was given an observation setting), the copy is its observation
  // instead (the plant state of an instance that does not observe), and a predicting instance b takes
  // age_b + d_b env steps: the actions applied since the observed record, then its queue (launch j: action
  // seq[b][j]; pred_len[b] = age_b + d_b).
  const float *qpos0 = B.qpos, *qvel0 = B.qvel, *warm0 = B.qacc_warmstart;
  const int32_t* cnt0 = B.counters;
  if (k.obs) {
    observe_kernel<<<ni, 128, 0, st>>>(p->dM, p->obs.d, p->ob, p->delay.d, Q.pending, env_step == 1, B.qpos, B.qvel,
                                       B.qacc_warmstart, B.counters, act, act_n1 * nu, P.qpos, P.qvel, P.warm, P.cnt);
    p->launches++;
    CUDA_OK(cudaGetLastError());
  } else if (k.npred > 0) {
    const size_t nq = p->hM.m.nq, nv = p->hM.m.nv;
    CUDA_OK(cudaMemcpyAsync(P.qpos, B.qpos, ni * nq * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaMemcpyAsync(P.qvel, B.qvel, ni * nv * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaMemcpyAsync(P.warm, B.qacc_warmstart, ni * nv * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaMemcpyAsync(P.cnt, B.counters, ni * 2 * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  }
  for (int j = 0; j < k.npred; ++j) {
    RolloutArgs A; memset(&A, 0, sizeof(A));
    A.qpos0 = P.qpos; A.qvel0 = P.qvel; A.warm0 = P.warm;
    A.counters_in = P.cnt; A.counters_out = P.cnt;
    A.nrows = ni; A.H = 1; A.mode = 0; A.rows_per_inst = 1;
    A.us = (k.obs ? p->ob.seq : Q.pending) + (size_t)j * nu; A.us_row = DIAL_MAXDELAY * nu;
    if (B.tasks) { A.tasks = B.tasks; A.task_rows = batched ? 1 : 0; }
    A.models = p->n_ens > 0 ? P.models : p->models.d;
    A.iter_lim = k.obs ? p->ob.len : Q.len; A.iter = j;
    A.qpos_out = P.qpos; A.qvel_out = P.qvel; A.warm_out = P.warm;
    A.terrain = planner_terrain;
    CUDA_OK(launch_rollout(p, A, 1, st));
  }
  if (k.planning()) { qpos0 = P.qpos; qvel0 = P.qvel; warm0 = P.warm; cnt0 = P.cnt; }
  // The info-only bars (qbar, qdbar, xbar; dial_core.py:133-135) are computed for EVERY iteration,
  // like the reference's scan does (the caller sees those of the last one), on a side branch of
  // the graph: the bars of iteration i read trajectory buffer i&1 and weights buffer i&1 while
  // iteration i+1 rolls into the other pair; iteration i+2 waits for them.
  const bool bars = B.qbar && B.qdbar && B.xbar;
  float* wts[2] = {p->weights, p->weights2};
  const size_t nw = (size_t)ni * (c.Ntotal + 1);   // weights of all instances
  for (int i = 0; i < n_diffuse; ++i) {
    const float* noise = B.noise + (size_t)i * n1;
    // rng split folded into the rollout (key = split(rng)[1]) and the fused update kernel (which also
    // advances rng); beyond 131072 samples the three-kernel sequence is kept
    const bool fused = c.Ntotal + 1 <= (1 << 17) && !getenv("DIAL_NO_FUSED_UPDATE");
    if (!fused) {
      mpc_split_kernel<<<1, 32, 0, st>>>(B.rng, p->mpc_key);
      p->launches++;
      CUDA_OK(cudaGetLastError());
    }
    if (bars && i >= 2) CUDA_OK(cudaStreamWaitEvent(st, p->ev_side[i & 1], 0));
    RolloutArgs A; memset(&A, 0, sizeof(A));
    A.qpos0 = qpos0; A.qvel0 = qvel0; A.warm0 = warm0; A.counters_in = cnt0;
    A.nrows = ni * K * (c.Nsample + 1); A.H = c.Hsample + 1; A.mode = 1;
    if (batched || p->n_ens > 0) A.rows_per_inst = K * (c.Nsample + 1);
    if (B.tasks) { A.tasks = B.tasks; A.task_rows = batched ? K * (c.Nsample + 1) : 0; }
    // the planner's models: the members (n_ens >= 1; the plan's model until one is set), else the instances'
    if (p->n_ens > 0) { A.rows_per_model = c.Nsample + 1; A.models = p->members.d; }
    else A.models = p->models.d;
    A.Ybar = Y[cur]; A.noise = noise;
    A.sched = p->sched.d; A.iter_lim = p->lims.d; A.iter = i;
    if (fused) A.rng_dev = B.rng; else A.key_dev = p->mpc_key;
    p->cur ^= 1;
    A.rews = K > 1 ? p->ens_rews : B.rews; A.q = p->traj_q[p->cur]; A.qd = p->traj_qd[p->cur]; A.xpos = p->traj_x[p->cur];
    A.dbg = p->dbg;
    A.terrain = planner_terrain;
    fill_xch(p, A);
    CUDA_OK(launch_rollout_any(p, A, st));
    if (K > 1) {   // each sample's score under its instance's risk measure (K = 1: the reward itself)
      const dim3 grid((c.Nsample + 1 + 255) / 256, ni);
      ensemble_reduce_kernel<<<grid, 256, 0, st>>>(p->ens_rews, p->risk.d, p->adapt.d, p->belief_w.d, K, c.Nsample + 1, B.rews,
                                                   p->lims.d, i);
      p->launches++;
      CUDA_OK(cudaGetLastError());
    }
    float* w = wts[i & 1];
    XchWait X = xch_wait_args(p, B.rews_all);
    if (fused) {
      int rc = launch_update(p, B.rews, w, X, B.rng, Y[cur], noise, Y[cur ^ 1], st, p->sched.d, p->lims.d, i,
                             wts[i > 0 ? (i - 1) & 1 : 0]);
      if (rc) return rc;
    } else {
      weights_kernel<<<1, 1024, 0, st>>>(B.rews, c.Ntotal + 1, c.temp_sample, w, X);
      p->launches++;
      CUDA_OK(cudaGetLastError());
      ybar_kernel<<<p->ybar_grid, YBAR_THREADS, 0, st>>>(w, nullptr, 0u, 0u, Y[cur], noise, c.Ntotal, n1, nu,
                                                         p->partial, p->counter, Y[cur ^ 1], p->mpc_key);
      p->launches++;
      CUDA_OK(cudaGetLastError());
    }
    cur ^= 1;
    if (bars) {
      CUDA_OK(cudaEventRecord(p->ev_main[i & 1], st));
      CUDA_OK(cudaStreamWaitEvent(p->side, p->ev_main[i & 1], 0));
      int rc = enqueue_trajbar(p, w, p->xch.on ? p->xch.rank : 0, B.qbar, B.qdbar, B.xbar, p->side, p->lims.d, i);
      if (rc) return rc;
      CUDA_OK(cudaEventRecord(p->ev_side[i & 1], p->side));
    }
  }
  if (cur != 0) CUDA_OK(cudaMemcpyAsync(Y[0], Y[1], (size_t)ni * n1 * nu * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (bars && n_diffuse > 0) {   // join the bars branch (both outstanding iterations)
    if (n_diffuse >= 2) CUDA_OK(cudaStreamWaitEvent(st, p->ev_side[(n_diffuse - 2) & 1], 0));
    CUDA_OK(cudaStreamWaitEvent(st, p->ev_side[(n_diffuse - 1) & 1], 0));
  }
  if (n_diffuse > 0 && wts[(n_diffuse - 1) & 1] != p->weights)   // p->weights always holds the last iteration's weights
    CUDA_OK(cudaMemcpyAsync(p->weights, p->weights2, nw * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

extern "C" int dial_mpc_step(dial_plan* p, int n_diffuse, int env_step, void* stream) {
  if (!p) return fail("dial_mpc_step: null plan");
  if (!p->mpc_bound) return fail("dial_mpc_step: call dial_mpc_bind first");
  if (n_diffuse < 0 || n_diffuse > 64) return fail("dial_mpc_step: n_diffuse out of range");
  if (env_step < 0 || env_step > 2) return fail("dial_mpc_step: env_step must be 0 (plan only), 1 (env step + shift) or 2 (shift only)");
  // batched plans use the fused update only (plan creation guarantees Nsample + 1 <= 2^17)
  if (p->n_inst > 1 && getenv("DIAL_NO_FUSED_UPDATE")) return fail("dial_mpc_step: batched plans need the fused update (unset DIAL_NO_FUSED_UPDATE)");
  if ((p->sched.d || p->lims.d) && getenv("DIAL_NO_FUSED_UPDATE"))
    return fail("dial_mpc_step: per-instance schedules and iteration limits need the fused update (unset DIAL_NO_FUSED_UPDATE)");
  // every instance with its own table has a row for each iteration it runs (the staging mirrors the device)
  for (int b = 0; p->sched.d && b < p->n_inst; ++b) {
    const InstSchedule& S = p->sched.h[b];
    const int runs = p->lims.d && p->lims.h[b] < n_diffuse ? p->lims.h[b] : n_diffuse;
    if (S.on && runs > S.n_rows)
      return fail("dial_mpc_step: instance " + std::to_string(b) + " runs " + std::to_string(runs) +
                  " diffusion iterations, its schedule has " + std::to_string(S.n_rows) + " rows");
  }
  cudaStream_t st = (cudaStream_t)stream;
  // the cached graphs replay the launch sequence of the last step's key: when the settings changed it, the next
  // use of each shape runs eagerly and the one after captures it again
  if (p->key != p->ran) drop_graphs(p);
  p->ran = p->key;
  dial_plan::MpcGraph* g = nullptr;
  for (auto& e : p->mpc_graphs) if (e.n_diffuse == n_diffuse && e.env_step == env_step) g = &e;
  if (!g) {
    // first use of this shape: run it eagerly (also configures the kernels' shared-memory limits)
    p->mpc_graphs.push_back({n_diffuse, env_step, 1, nullptr, 0});
    return mpc_enqueue(p, p->ran, n_diffuse, env_step, st);
  }
  if (!g->exec) {
    if (getenv("DIAL_NO_GRAPH")) return mpc_enqueue(p, p->ran, n_diffuse, env_step, st);
    // second use: capture the same sequence into a graph, then replay it from now on
    cudaStream_t cs;
    CUDA_OK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    const int64_t l0 = p->launches;
    cudaError_t e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
    if (e != cudaSuccess) { cudaStreamDestroy(cs); CUDA_OK(e); }
    int rc = mpc_enqueue(p, p->ran, n_diffuse, env_step, cs);
    cudaGraph_t graph = nullptr;
    e = cudaStreamEndCapture(cs, &graph);
    cudaStreamDestroy(cs);
    g->launches = p->launches - l0;
    p->launches = l0;
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    CUDA_OK(e);
    e = cudaGraphInstantiate(&g->exec, graph, 0);
    cudaGraphDestroy(graph);
    CUDA_OK(e);
  }
  CUDA_OK(cudaGraphLaunch(g->exec, st));
  p->launches += g->launches;
  return 0;
}

extern "C" void dial_key_split(const uint32_t key[2], uint32_t out0[2], uint32_t out1[2]) {
  // jax.random.split(key, 2), legacy layout: counters [0,1,2,3] -> halves (0,1) | (2,3)
  uint32_t a0 = 0, b0 = 2, a1 = 1, b1 = 3;
  threefry2x32(key[0], key[1], a0, b0);
  threefry2x32(key[0], key[1], a1, b1);
  out0[0] = a0; out0[1] = a1; out1[0] = b0; out1[1] = b1;
}

extern "C" int dial_solver_variant(const dial_model_desc* model) {
  if (!model) return fail("null descriptor");
  DevModel* D = new (std::nothrow) DevModel();
  if (!D) return fail("out of memory");
  std::string err;
  int v = -1;
  if (!derive_model(*model, *D, err)) g_err = err;
  else if ((v = star_variant(*D)) < 0) g_err = "this build instantiates the dense (elliptic) solver path for nv = " DIAL_STR(DIAL_DENSE_NV) " only (custom builds: dial_mpc_b200.custom compiles it for the model's nv)";
  delete D;
  return v;
}

extern "C" const char* dial_plan_rollout_kernel(const dial_plan* p) {
  return p ? p->kernels.name : "";
}

extern "C" const char* dial_custom_reward_id(void) {
#if defined(DIAL_CUSTOM_REWARD_FILE) && defined(DIAL_CUSTOM_REWARD_ID)
  return DIAL_STR(DIAL_CUSTOM_REWARD_ID);
#elif defined(DIAL_CUSTOM_REWARD_FILE)
  return "custom";
#else
  return "";
#endif
}

// ---- in-run fp32 peak (roofline denominator): independent FFMA chains at full occupancy ------
__global__ void __launch_bounds__(1024) fp32_peak_kernel(float* out, int iters, float a, float b) {
  float x[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = (float)(threadIdx.x + i) * 1e-3f;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int r = 0; r < 16; ++r) {
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] = fmaf(x[i], a, b);
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += x[i];
  if (s == 123.456f) out[0] = s;   // never true: keeps the chains alive
}

extern "C" int dial_fp32_peak(int iters, float* tflops_out) {
  if (!tflops_out || iters < 1) return fail("dial_fp32_peak: bad argument");
  int dev = 0, sms = 0;
  CUDA_OK(cudaGetDevice(&dev));
  CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  float* d = nullptr;
  CUDA_OK(cudaMalloc(&d, sizeof(float)));
  cudaEvent_t e0, e1;
  CUDA_OK(cudaEventCreate(&e0));
  CUDA_OK(cudaEventCreate(&e1));
  const int grid = sms * 2;
  fp32_peak_kernel<<<grid, 1024>>>(d, 64, 0.999f, 1e-3f);   // warm-up
  float best = 0.f;
  for (int rep = 0; rep < 3; ++rep) {
    cudaEventRecord(e0);
    fp32_peak_kernel<<<grid, 1024>>>(d, iters, 0.999f, 1e-3f);
    cudaEventRecord(e1);
    cudaError_t e = cudaEventSynchronize(e1);
    if (e != cudaSuccess) { cudaFree(d); return fail(std::string("fp32 peak kernel: ") + cudaGetErrorString(e)); }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    const double flop = 2.0 * 8 * 16 * (double)iters * 1024.0 * grid;
    const float tf = (float)(flop / (ms * 1e-3) / 1e12);
    best = tf > best ? tf : best;
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d);
  *tflops_out = best;
  return 0;
}

extern "C" int64_t dial_launch_count(const dial_plan* p) { return p ? p->launches : 0; }
extern "C" int dial_rollout_wpc(const dial_plan* p, int nrows) { return (p && nrows > 0) ? default_wpc(p, nrows) : 0; }

extern "C" int dial_debug_counters(dial_plan* p, float out[8]) {
  if (!p || !p->dbg) return fail("debug counters are off (set DIAL_DEBUG_COUNTERS=1 before dial_plan_create)");
  CUDA_OK(cudaMemcpy(out, p->dbg, 8 * sizeof(float), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemset(p->dbg, 0, 8 * sizeof(float)));
  return 0;
}
