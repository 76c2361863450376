// libmwb200: batched Meta-World step engine for H100 (sm_90a).  C ABI: include/metaworld_b200.h.
//
// One warp = one environment for a whole env step: 5 x (forward dynamics + semi-implicit Euler), one more
// forward pass, observation, reward/info, time-limit / success termination and autoreset (SAME_STEP, NEXT_STEP or none), with the
// per-env state making a single 512-byte round trip to HBM (coalesced 128-bit loads/stores).  One CTA = WARPS_PER_BLOCK warps
// that share one task model; the ~10 KB model blob is staged into shared memory with a TMA bulk copy
// (cp.async.bulk + mbarrier).  There is no CPU fallback: every entry point launches CUDA kernels or fails.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "../../include/metaworld_b200.h"
#include "mw_tasks.cuh"
#include "mw_policies.cuh"

#ifndef WARPS_PER_BLOCK
#define WARPS_PER_BLOCK 7
#endif
#define BLOCK_THREADS (WARPS_PER_BLOCK * 32)
#define MW_ENVPROF_W 20       // words per env in the optional per-env profile record (mw_get_env_profile)

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(MW_ERR_CUDA, std::string(#x ": ") + cudaGetErrorString(e_)); } while (0)

struct EngineDev {
  const unsigned char* models; int model_stride;     // MwModel blobs (stride multiple of 16)
  const MwTaskConst* taskconsts;
  const float* const* meshverts;                     // [n_models] device pointers
  MwEnvState* state; MwSnapshot* snaps;
  const int* goal_first; const int* goal_count;      // device sampler ranges (may be NULL)
  int* diag;                                         // [n_envs][3]: contacts dropped, solver iterations, MW_FAULT_* bits (OR)
  EpaWs* epa;                                        // GJK/EPA polytope workspace, one per warp slot (global memory, see scratch_slot)
  WarpSpill* spill;                                  // overflow contacts / constraint rows, one block per warp slot (global memory)
  int slot_by_sm;                                    // warp slots are numbered by SM (one resident CTA per SM) instead of by CTA
  unsigned long long* prof;                          // [16] summed cycle / event counters (mw_get_profile)
  unsigned long long* model_cycles;                  // [n_models][2]: warp cycles, env steps (drives mw_rebalance)
  unsigned* env_cost;                                // [n_envs] solver work of each env's previous step (orders the envs of a model, k_order_envs)
  unsigned* env_cycles;                              // [n_envs] cycles each env's warp spent in its previous k_step = duration of its CTA (orders the CTAs, k_order_blocks)
  float4* sep_hint;                                  // [n_envs][MW_NCONV] separating-axis hints of the general convex pairs (k_step only; mw_collide)
  unsigned* env_prof;                                // optional [n_envs][16] per-env phase cycles / event counts of the last step (mw_set_profiling)
  int n_envs, max_steps, terminate_on_success; unsigned long long seed;
  int autoreset_mode;                                // MW_AUTORESET_* (mw_set_autoreset_mode)
};

// The per-warp global scratch (EPA polytope, overflow rows) is addressed by SM, not by CTA, when at most one CTA fits an SM:
// n_SM x WARPS_PER_BLOCK blocks (132 SMs on an H100) that successive CTAs of an SM reuse stay resident in L2, whereas one block per launched warp
// (4200 x 10.7 KB for 4096 envs) is a stream of first-touch lines that all end up in DRAM.
DEV unsigned mw_smid() { unsigned r; asm volatile("mov.u32 %0, %%smid;" : "=r"(r)); return r; }
DEV size_t scratch_slot(const EngineDev& e, int warp) { return (size_t)(e.slot_by_sm ? mw_smid() : blockIdx.x) * WARPS_PER_BLOCK + warp; }
__global__ void k_nsmid(unsigned* out) { unsigned r; asm volatile("mov.u32 %0, %%nsmid;" : "=r"(r)); *out = r; }

// ---------------------------------------------------------------- shared memory carve-up
struct BlockShared {
  alignas(16) unsigned char model[(sizeof(MwModel) + 15) / 16 * 16];
  MwTaskConst tc;
  CtaShare cs;
  alignas(8) unsigned long long bar;
};
struct WarpShared {
  WarpScratch w;
  alignas(16) MwEnvState es;
  float obs[40]; float info[8];
};
static size_t smem_bytes() { return sizeof(BlockShared) + WARPS_PER_BLOCK * sizeof(WarpShared) + 16; }

DEV unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
// TMA bulk copy global -> shared with mbarrier completion (SASS: UBLKCP / SYNCS)
DEV void stage_model(BlockShared* bs, const unsigned char* src, unsigned bytes, const MwTaskConst* tc_src) {
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bs->bar)));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bs->bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(bs->model)), "l"(src), "r"(bytes), "r"(smem_u32(&bs->bar)) : "memory");
  }
  // the small task-constant record rides along with ordinary loads
  for (int i = threadIdx.x; i < (int)(sizeof(MwTaskConst) / 4); i += blockDim.x) ((int*)&bs->tc)[i] = ((const int*)tc_src)[i];
  unsigned ok = 0;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(smem_u32(&bs->bar)), "r"(0u) : "memory");
  } while (!ok);
  __syncthreads();
}

// wires a warp into its CTA's convex-pair queue (mw_physics.cuh: CtaShare); visible to the other warps after the first PHASE_SYNC
// `sep`: the env's row of the separating-axis hint table (k_step); the other kernels run without hints
DEV void join_cta(BlockShared* bs, WarpShared* wsa, WarpScratch* w, int warp, int live_warps, float4* sep = nullptr) {
  if (threadIdx.x == 0) { bs->cs.q_head = 0; bs->cs.nwarp = live_warps; bs->cs.peer_stride = (int)sizeof(WarpShared); bs->cs.peer0 = (unsigned char*)wsa; }
  if ((threadIdx.x & 31) == 0) { w->cta = &bs->cs; w->warp_in_cta = warp; w->ncand = 0; w->prof_on = 0; w->nblk1 = mw_tree_split((const MwModel*)bs->model); w->sep = sep; }
#ifdef MW_CHOL_ONE_CHAIN     /* A/B switch: never split the factorisation */
  if ((threadIdx.x & 31) == 0) w->nblk1 = ((const MwModel*)bs->model)->nv;
#endif
  __syncwarp();
}
__device__ void eng_forward(const TaskCtx& c, int lane) { mw_forward(c.m, c.meshvert, c.w, lane); }
__device__ void eng_sim(const TaskCtx& c, int nstep, int lane) {
  for (int s = 0; s < nstep; s++) { mw_forward(c.m, c.meshvert, c.w, lane); mw_euler(c.m, c.w, lane); }
}

// ---------------------------------------------------------------- state <-> scratch
DEV void load_env(WarpShared* ws, const MwEnvState* src, int lane) {
  ((float4*)&ws->es)[lane] = ((const float4*)src)[lane];     // 32 lanes x 16 B = the whole 512 B record
  SYNCW();
  WarpScratch* w = &ws->w;
  if (lane < MW_MAXNQ) { w->qposd[lane] = ws->es.qpos[lane]; w->qpos[lane] = (real)w->qposd[lane]; }
  if (lane < MW_MAXDOF) { w->qvel[lane] = ws->es.qvel[lane]; w->warm[lane] = ws->es.warm[lane]; }
  if (lane < 3) { w->mocap_pos[lane] = ws->es.mocap_pos[lane]; w->shift[lane] = ws->es.shift[lane]; }
  if (lane == 0) { w->mocap_quat[0] = 1; w->mocap_quat[1] = 0; w->mocap_quat[2] = 1; w->mocap_quat[3] = 0; w->ctrl[0] = w->ctrl[1] = 0; }
  SYNCW();
}
DEV void store_env(WarpShared* ws, MwEnvState* dst, int lane) {
  WarpScratch* w = &ws->w;
  if (lane < MW_MAXNQ) ws->es.qpos[lane] = w->qposd[lane];
  if (lane < MW_MAXDOF) { ws->es.qvel[lane] = (float)w->qvel[lane]; ws->es.warm[lane] = (float)w->warm[lane]; }
  if (lane < 3) { ws->es.mocap_pos[lane] = (float)w->mocap_pos[lane]; ws->es.shift[lane] = (float)w->shift[lane]; }
  SYNCW();
  ((float4*)dst)[lane] = ((const float4*)&ws->es)[lane];
}

// observation assembly (sawyer_xyz_env.py:475-527 + clip :623-628); lane 0
DEV void make_obs(const TaskCtx& c, float* obs, bool clip = true) {   // reset() returns the observation unclipped (:664-682)
  real cur[18];
  mw_frame_pos(c.m, c.w, F_HAND, cur);
  real a[3], b[3]; mw_frame_pos(c.m, c.w, F_RCLAW, a); mw_frame_pos(c.m, c.w, F_LCLAW, b);
  cur[3] = fmin(fmax(dist3(a, b) / (real)0.1, (real)0), (real)1);
  task_obs_objects(c, cur + 4);
  const real hlo[3] = {(real)-0.525, (real)0.348, (real)-0.0525}, hhi[3] = {(real)0.525, (real)1.025, (real)0.7};
  for (int i = 0; i < 18; i++) {
    real v = cur[i], pv = c.s->prev_obs[i];
    if (clip && i < 3) { v = fmin(fmax(v, hlo[i]), hhi[i]); pv = fmin(fmax(pv, hlo[i]), hhi[i]); }
    if (clip && i == 3) { v = fmin(fmax(v, (real)-1), (real)1); pv = fmin(fmax(pv, (real)-1), (real)1); }
    obs[i] = (float)v; obs[18 + i] = (float)pv;
    c.s->prev_obs[i] = (float)cur[i];
  }
  for (int i = 0; i < 3; i++) {
    real g = c.s->partially_observable != 0.f ? (real)0 : (clip ? fmin(fmax((real)c.s->target[i], (real)c.tc->goal_lo[i]), (real)c.tc->goal_hi[i]) : (real)c.s->target[i]);
    obs[36 + i] = (float)g;
  }
}

DEV unsigned long long mix64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31);
}
// device task sampler: the snapshot env `env` restarts from after its episode number `episode` (mw_set_goal_sets)
DEV int sample_snapshot(const EngineDev& e, int env, float episode) {
  unsigned long long h = mix64(e.seed ^ mix64(((unsigned long long)env << 32) | (unsigned)(int)episode));
  return e.goal_first[env] + (int)(h % (unsigned long long)e.goal_count[env]);
}

// ---------------------------------------------------------------- kernels
// DEFERRED = false: SAME_STEP autoreset; true: NEXT_STEP or DISABLED (e.autoreset_mode tells which).  Two instantiations,
// so that the default path carries none of the code of the other modes (the kernel is bound by instruction fetch)
template <bool DEFERRED>
__global__ void __launch_bounds__(BLOCK_THREADS, 1)
k_step(EngineDev e, const int* __restrict__ block_order, const int* __restrict__ block_model, const int* __restrict__ block_start, const int* __restrict__ block_count,
       const int* __restrict__ perm, const float* __restrict__ actions, float* __restrict__ obs_out, int obs_stride,
       float* __restrict__ reward, unsigned char* __restrict__ terminated, unsigned char* __restrict__ truncated,
       float* __restrict__ info_out, int info_stride, float* __restrict__ final_obs, float* __restrict__ final_info, const int* __restrict__ next_snapshot,
       const int* __restrict__ block_live) {
  extern __shared__ __align__(16) unsigned char smem[];
  BlockShared* bs = (BlockShared*)smem;
  WarpShared* wsa = (WarpShared*)(smem + sizeof(BlockShared));
  const int blk = block_order[blockIdx.x];             // launch slot -> CTA work item (costliest first, see k_order_*)
  if (block_live && !block_live[blk]) return;          // the other decomposition of this model's head is running (k_order_blocks)
  const int mi = block_model[blk];
  stage_model(bs, e.models + (size_t)mi * e.model_stride, (unsigned)sizeof(bs->model), e.taskconsts + mi);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp >= block_count[blk]) return;
  const int env = perm[block_start[blk] + warp];
  WarpShared* ws = wsa + warp;
  ws->w.epa = e.epa + scratch_slot(e, warp);
  ws->w.sp = e.spill + scratch_slot(e, warp);
  WarpScratch* w = &ws->w;
  join_cta(bs, wsa, w, warp, block_count[blk], e.sep_hint + (size_t)env * MW_NCONV);
  const MwModel* m = (const MwModel*)bs->model;
  load_env(ws, e.state + env, lane);
  // NEXT_STEP / DISABLED: an env whose episode ended in the previous call still runs its physics below, so that its warp
  // takes part in the CTA's phase barriers, and the result is discarded in the tail (restart, or nothing at all)
  const bool ended = DEFERRED && ws->es.ended != 0.f;
  if (lane < 16) w->prof[lane] = 0;
  if (lane == 0) { w->fault = 0; w->prof_on = e.prof != nullptr; }
  SYNCW();
  const long long t_begin = MW_CLK(w);
  const long long t_cta = e.env_cycles ? mw_clock() : 0ll;
  real act[4];
  for (int i = 0; i < 4; i++) act[i] = fmin(fmax((real)actions[4 * env + i], (real)-1), (real)1);
  TaskCtx c; c.m = m; c.tc = &bs->tc; c.w = w; c.s = &ws->es; c.action = act; c.meshvert = e.meshverts[mi];
  // set_xyz_action (sawyer_xyz_env.py:320-336) + ctrl = [a3, -a3] (:595)
  if (lane < 3) w->mocap_pos[lane] = fmin(fmax(w->mocap_pos[lane] + act[lane] * (real)0.01, (real)bs->tc.mocap_lo[lane]), (real)bs->tc.mocap_hi[lane]);
  if (lane == 0) { w->ctrl[0] = (real)actions[4 * env + 3]; w->ctrl[1] = -(real)actions[4 * env + 3]; }
  SYNCW();
  int iters = 0, dropped = 0, ncon_max = 0, nefc_max = 0, solver_work = 0, cand_total = 0;
  for (int s = 0; s < 5; s++) {
    mw_forward(m, c.meshvert, w, lane);
    iters += w->solver_iter; dropped += w->ncon_dropped; ncon_max = max(ncon_max, w->ncon); nefc_max = max(nefc_max, w->nefc);
    solver_work += (w->solver_iter + 1) * (w->nefc + 4 * w->ncon + 24); cand_total += w->ncand;
    mw_euler(m, w, lane);
  }
  // mj_forward (sawyer_xyz_env.py:620): full pass only where the reward reads contact forces (same task for the whole CTA)
  if (task_needs_contact_forces(bs->tc.task_id)) {
    mw_forward(m, c.meshvert, w, lane);
    iters += w->solver_iter; dropped += w->ncon_dropped; ncon_max = max(ncon_max, w->ncon); nefc_max = max(nefc_max, w->nefc);
    solver_work += (w->solver_iter + 1) * (w->nefc + 4 * w->ncon + 24); cand_total += w->ncand;
  } else mw_forward_kinematics_only(m, w, lane);
  bool done = false;
  const long long t_phys = MW_CLK(w);
  if (lane == 0) {
    ws->es.path_len += 1.f;
    task_live_update(c);
    make_obs(c, ws->obs);
    real obsr[39]; for (int i = 0; i < 39; i++) obsr[i] = ws->obs[i];
    real rew, inf[INFO_N];
    real raw_act[4]; for (int i = 0; i < 4; i++) raw_act[i] = actions[4 * env + i];
    c.action = raw_act;
    task_reward(c, obsr, &rew, inf);
    for (int i = 0; i < INFO_N; i++) ws->info[i] = (float)inf[i];
    ws->es.ep_return += (float)rew;
    bool trunc = ws->es.path_len >= (float)e.max_steps;
    bool term = e.terminate_on_success && inf[INFO_SUCCESS] == (real)1;
    ws->info[7] = (term || trunc) ? 1.f : 0.f;
    if (!ended) {
      reward[env] = (float)rew; terminated[env] = term; truncated[env] = trunc;
      if (info_stride >= 9) { info_out[(size_t)env * info_stride + 7] = (float)rew; info_out[(size_t)env * info_stride + 8] = (float)((int)term + 2 * (int)trunc); }   // packed record: one D2H copy
      { bool fin = isfinite((float)rew); for (int i = 0; i < 39; i++) fin = fin && isfinite(ws->obs[i]); if (!fin) w->fault |= MW_FAULT_NONFINITE; }
      e.diag[3 * env] += dropped; e.diag[3 * env + 1] += iters; e.diag[3 * env + 2] |= w->fault;
    } else if (e.autoreset_mode == MW_AUTORESET_DISABLED) e.diag[3 * env + 2] |= MW_FAULT_STEP_AFTER_END;   // the discarded pass reports nothing else
    w->prof[7] = MW_CLK(w) - t_phys; w->prof[8] = MW_CLK(w) - t_begin;
    // launch-order key: the cycles this env spent in its constraint solver + constraint assembly.  The whole-step time
    // is the same for all warps of a CTA (they wait for each other at every phase boundary) and would keep light envs
    // glued to the heavy one they were once grouped with; the collision phase is shared across the CTA (CtaShare); the
    // other phases cost the same for every env of a model.  What is left to group by is the solver.
    const long long own = w->prof[8] - w->prof[12];
    // (a work estimate from counters rather than the cycle clock: Newton iterations weighted by the rows they touch)
    e.env_cost[env] = (unsigned)solver_work;
    if (e.env_cycles) { long long d = mw_clock() - t_cta; e.env_cycles[env] = (unsigned)(d > 0xFFFFFFFFll ? 0xFFFFFFFFll : d); }
    w->prof[6] = own - w->prof[7] - (w->prof[0] + w->prof[1] + w->prof[3] + w->prof[4] + w->prof[5]);   // euler + glue
  }
  SYNCW();
  if (e.prof) {     // profiling runs only (mw_set_profiling): summed phase counters, per-model cost, per-env record
    if (lane < 15) atomicAdd(e.prof + lane, (unsigned long long)w->prof[lane]);
    if (lane == 0 && e.model_cycles) { atomicAdd(e.model_cycles + 2 * mi, (unsigned long long)w->prof[8]); atomicAdd(e.model_cycles + 2 * mi + 1, 1ull); }
    if (e.env_prof) {
      if (lane < 13) e.env_prof[MW_ENVPROF_W * env + lane] = (unsigned)(w->prof[lane] > 0xFFFFFFFFll ? 0xFFFFFFFFll : w->prof[lane]);
      if (lane == 13) e.env_prof[MW_ENVPROF_W * env + 13] = (unsigned)iters;
      if (lane == 14) e.env_prof[MW_ENVPROF_W * env + 14] = (unsigned)ncon_max;
      if (lane == 15) e.env_prof[MW_ENVPROF_W * env + 15] = (unsigned)nefc_max;
      if (lane == 16) e.env_prof[MW_ENVPROF_W * env + 16] = (unsigned)blockIdx.x;
      if (lane == 17) e.env_prof[MW_ENVPROF_W * env + 17] = (unsigned)cand_total;      // convex candidate pairs this env queued
      if (lane == 18 || lane == 19) e.env_prof[MW_ENVPROF_W * env + lane] = (unsigned)w->prof[lane - 5];   // hint tests / rejections by this warp
    }
  }
  done = ws->info[7] != 0.f;
  if (ended) {
    if (e.autoreset_mode == MW_AUTORESET_DISABLED) return;      // state record and output rows stay as they are
    // NEXT_STEP, the call after the terminal step: the action is ignored, the env restarts and reports the reset
    // observation with reward 0, no done flags and an all-zero info row
    if (lane < INFO_N) info_out[(size_t)env * info_stride + lane] = 0.f;
    if (lane == 0) {
      reward[env] = 0.f; terminated[env] = 0; truncated[env] = 0;
      if (info_stride >= 9) { info_out[(size_t)env * info_stride + 7] = 0.f; info_out[(size_t)env * info_stride + 8] = 0.f; }
    }
  } else {
    if (lane < INFO_N) info_out[(size_t)env * info_stride + lane] = ws->info[lane];
    if (!done || DEFERRED) {
      // NEXT_STEP / DISABLED terminal step: the terminal observation goes to obs, the env is marked and restarts later;
      // the episode return still goes to final_info column 7 (episode statistics)
      if (DEFERRED && done) {
        if (final_info && lane == 7) final_info[(size_t)env * 8 + 7] = ws->es.ep_return;
        if (lane == 0) ws->es.ended = 1.f;
      }
      if (lane == 0) ws->es.gripper_ctrl = actions[4 * env + 3];   // data.ctrl of this state (k_query's contact forces)
      for (int i = lane; i < 39; i += 32) obs_out[(size_t)env * obs_stride + i] = ws->obs[i];
      store_env(ws, e.state + env, lane);
      return;
    }
    // SAME_STEP autoreset: report the terminal transition, restart from a cached episode-start snapshot
    if (final_obs) for (int i = lane; i < 39; i += 32) final_obs[(size_t)env * obs_stride + i] = ws->obs[i];
    if (final_info) { if (lane < INFO_N) final_info[(size_t)env * 8 + lane] = ws->info[lane]; if (lane == 7) final_info[(size_t)env * 8 + 7] = ws->es.ep_return; }
  }
  {
    // restart (same snapshot choice and episode count in both modes, so NEXT_STEP runs the goal sequence of SAME_STEP)
    const int snap = next_snapshot ? next_snapshot[env] : sample_snapshot(e, env, ws->es.episode);
    float episode = ws->es.episode + 1.f;
    const MwSnapshot* sp = e.snaps + snap;
    float4 v = ((const float4*)&sp->st)[lane];
    SYNCW();
    ((float4*)&ws->es)[lane] = v;
    SYNCW();
    if (lane == 0) { ws->es.episode = episode; ws->es.snapshot = (float)snap; ws->es.ep_return = 0.f; ws->es.path_len = 0.f; }
    SYNCW();
    ((float4*)(e.state + env))[lane] = ((const float4*)&ws->es)[lane];
    for (int i = lane; i < 39; i += 32) obs_out[(size_t)env * obs_stride + i] = sp->obs[i];
  }
}

// builds episode-start snapshots: exact reset() sequence of the reference (reset_model, mj_resetData, reset_model)
__global__ void __launch_bounds__(BLOCK_THREADS, 1)
k_snapshot(EngineDev e, const int* __restrict__ block_model, const int* __restrict__ block_start, const int* __restrict__ block_count,
           const int* __restrict__ perm, const double* __restrict__ rand_vec, const double* __restrict__ rand_vec_pass1, const unsigned char* __restrict__ partial, int snap_base) {
  extern __shared__ __align__(16) unsigned char smem[];
  BlockShared* bs = (BlockShared*)smem;
  WarpShared* wsa = (WarpShared*)(smem + sizeof(BlockShared));
  const int mi = block_model[blockIdx.x];
  stage_model(bs, e.models + (size_t)mi * e.model_stride, (unsigned)sizeof(bs->model), e.taskconsts + mi);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp >= block_count[blockIdx.x]) return;
  const int item = perm[block_start[blockIdx.x] + warp];
  WarpShared* ws = wsa + warp;
  ws->w.epa = e.epa + scratch_slot(e, warp);
  ws->w.sp = e.spill + scratch_slot(e, warp);
  WarpScratch* w = &ws->w;
  join_cta(bs, wsa, w, warp, block_count[blockIdx.x]);
  const MwModel* m = (const MwModel*)bs->model;
  const double* rv2 = rand_vec + 6 * item;
  const double* rv1 = rand_vec_pass1 ? rand_vec_pass1 + 6 * item : rv2;   // an unfrozen rand_vec draws once per reset_model pass
  real act[4] = {0, 0, 0, 0};
  TaskCtx c; c.m = m; c.tc = &bs->tc; c.w = w; c.s = &ws->es; c.action = act; c.meshvert = e.meshverts[mi];
  for (int i = lane; i < 128; i += 32) ((float*)&ws->es)[i] = 0.f;
  if (lane < 3) w->shift[lane] = 0;
  SYNCW();
  for (int pass = 0; pass < 2; pass++) {
    {
      // mj_resetData (pass 0: a freshly constructed env is in the same state)
      if (lane < MW_MAXNQ) QSET(w, lane, lane < m->nq ? m->qpos0d[lane] : 0.0);
      if (lane < MW_MAXDOF) { w->qvel[lane] = 0; w->warm[lane] = 0; }
      if (lane < 3) w->mocap_pos[lane] = m->mocap_pos0[lane];
      if (lane < 4) w->mocap_quat[lane] = m->mocap_quat0[lane];
      if (lane < 2) w->ctrl[lane] = 0;
      SYNCW();
    }
    // _reset_hand (sawyer_xyz_env.py:684-695)
    for (int k = 0; k < 50; k++) {
      if (lane < 3) w->mocap_pos[lane] = bs->tc.hand_init[lane];
      if (lane == 0) { w->mocap_quat[0] = 1; w->mocap_quat[1] = 0; w->mocap_quat[2] = 1; w->mocap_quat[3] = 0; w->ctrl[0] = -1; w->ctrl[1] = 1; }
      SYNCW();
      eng_sim(c, 5, lane);
    }
    if (lane == 0) { real t[3]; tcp_center(c, t); for (int i = 0; i < 3; i++) ws->es.init_tcp[i] = (float)t[i]; }
    SYNCW();
    task_reset_model(c, pass == 0 ? rv1 : rv2, lane);
    SYNCW();
  }
  if (lane == 0) {
    ws->es.partially_observable = partial[item] ? 1.f : 0.f;
    make_obs(c, ws->obs, false);                       // _get_obs() of pass 2, not clipped
    for (int i = 0; i < 18; i++) { ws->obs[18 + i] = ws->obs[i]; }   // reset(): obs[18:36] = obs[:18]  (:679-680)
    ws->es.path_len = 0.f; ws->es.episode = 0.f; ws->es.ep_return = 0.f; ws->es.snapshot = (float)(snap_base + item);
    ws->es.gripper_ctrl = -1.f;                        // _reset_hand leaves ctrl = [-1, 1]
  }
  SYNCW();
  if (lane < 3) ws->es.shift[lane] = (float)w->shift[lane];
  SYNCW();
  MwSnapshot* sp = e.snaps + snap_base + item;
  store_env(ws, &sp->st, lane);
  for (int i = lane; i < 39; i += 32) sp->obs[i] = ws->obs[i];
}

__global__ void k_reset(EngineDev e, int n, const int* __restrict__ env_ids, const int* __restrict__ snapshot_ids,
                        float* __restrict__ obs, int obs_stride) {
  int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (gw >= n) return;
  int env = env_ids ? env_ids[gw] : gw;
  const MwSnapshot* sp = e.snaps + snapshot_ids[gw];
  float4 v = ((const float4*)&sp->st)[lane];
  ((float4*)(e.state + env))[lane] = v;
  if (lane == 0) e.state[env].snapshot = (float)snapshot_ids[gw];
  for (int i = lane; i < 39; i += 32) obs[(size_t)gw * obs_stride + i] = sp->obs[i];
}

// partial reset, one warp per env: envs with mask[env] set restart from snapshot_ids[env] (NULL: the device sampler's draw)
// and count one more episode, as the autoreset does; obs row env is written, the other rows are left alone
__global__ void k_reset_masked(EngineDev e, const unsigned char* __restrict__ mask, const int* __restrict__ snapshot_ids,
                               float* __restrict__ obs, int obs_stride) {
  const int env = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (env >= e.n_envs || !mask[env]) return;
  const float episode = e.state[env].episode;
  const int snap = snapshot_ids ? snapshot_ids[env] : sample_snapshot(e, env, episode);
  const MwSnapshot* sp = e.snaps + snap;
  float4 v = ((const float4*)&sp->st)[lane];
  __syncwarp();                                        // every lane has read `episode` before the record is overwritten
  ((float4*)(e.state + env))[lane] = v;
  __syncwarp();
  if (lane == 0) { e.state[env].episode = episode + 1.f; e.state[env].snapshot = (float)snap; }
  for (int i = lane; i < 39; i += 32) obs[(size_t)env * obs_stride + i] = sp->obs[i];
}

__global__ void __launch_bounds__(BLOCK_THREADS, 1)
k_substeps(EngineDev e, const int* __restrict__ block_model, const int* __restrict__ block_start, const int* __restrict__ block_count,
           const int* __restrict__ perm, int nstep, float c0, float c1, float* __restrict__ dump) {
  extern __shared__ __align__(16) unsigned char smem[];
  BlockShared* bs = (BlockShared*)smem;
  WarpShared* wsa = (WarpShared*)(smem + sizeof(BlockShared));
  const int mi = block_model[blockIdx.x];
  stage_model(bs, e.models + (size_t)mi * e.model_stride, (unsigned)sizeof(bs->model), e.taskconsts + mi);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp >= block_count[blockIdx.x]) return;
  const int env = perm[block_start[blockIdx.x] + warp];
  WarpShared* ws = wsa + warp;
  ws->w.epa = e.epa + scratch_slot(e, warp);
  ws->w.sp = e.spill + scratch_slot(e, warp);
  join_cta(bs, wsa, &ws->w, warp, block_count[blockIdx.x]);
  const MwModel* m = (const MwModel*)bs->model;
  load_env(ws, e.state + env, lane);
  if (lane == 0) { ws->w.ctrl[0] = c0; ws->w.ctrl[1] = c1; }
  SYNCW();
  for (int s = 0; s < nstep; s++) { mw_forward(m, e.meshverts[mi], &ws->w, lane); mw_euler(m, &ws->w, lane); }
  if (dump) {   // debug: one forward pass, then dump contacts [env][MW_MAXCON][12] and qacc [env][MW_MAXDOF] after them
    mw_forward(m, e.meshverts[mi], &ws->w, lane);
    float* d = dump + (size_t)env * (MW_MAXCON * 12 + MW_MAXDOF + 4);
    for (int c = lane; c < MW_MAXCON; c += 32) {
      const Contact* k = mw_con(&ws->w, c);
      bool ok = c < ws->w.ncon;
      d[12 * c + 0] = ok ? (float)k->dist : 0.f;
      for (int i = 0; i < 3; i++) { d[12 * c + 1 + i] = ok ? (float)k->pos[i] : 0.f; d[12 * c + 4 + i] = ok ? (float)k->frame[i] : 0.f; }
      d[12 * c + 7] = ok ? (float)m->geom_srcid[k->g1] : -1.f; d[12 * c + 8] = ok ? (float)m->geom_srcid[k->g2] : -1.f;
      d[12 * c + 9] = ok ? (float)k->fn : 0.f; d[12 * c + 10] = ok ? (float)k->dim : 0.f; d[12 * c + 11] = ok ? (float)k->row : -1.f;
    }
    if (lane < MW_MAXDOF) d[MW_MAXCON * 12 + lane] = (float)ws->w.qacc[lane];
    if (lane == 0) { d[MW_MAXCON * 12 + MW_MAXDOF] = (float)ws->w.ncon; d[MW_MAXCON * 12 + MW_MAXDOF + 1] = (float)ws->w.nefc; d[MW_MAXCON * 12 + MW_MAXDOF + 2] = (float)ws->w.solver_iter; }
    return;
  }
  store_env(ws, e.state + env, lane);
}

// evaluate_state (sawyer_xyz_env.py:644-656 + the task's compute_reward): reward / info of the CURRENT state for a given
// (obs, action); one forward pass to rebuild poses and contact forces, nothing is written back to the state
__global__ void __launch_bounds__(BLOCK_THREADS, 1)
k_evaluate(EngineDev e, const int* __restrict__ block_model, const int* __restrict__ block_start, const int* __restrict__ block_count,
           const int* __restrict__ perm, const float* __restrict__ actions, const float* __restrict__ obs_in, int obs_stride, float* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem[];
  BlockShared* bs = (BlockShared*)smem;
  WarpShared* wsa = (WarpShared*)(smem + sizeof(BlockShared));
  const int mi = block_model[blockIdx.x];
  stage_model(bs, e.models + (size_t)mi * e.model_stride, (unsigned)sizeof(bs->model), e.taskconsts + mi);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp >= block_count[blockIdx.x]) return;
  const int env = perm[block_start[blockIdx.x] + warp];
  WarpShared* ws = wsa + warp;
  ws->w.epa = e.epa + scratch_slot(e, warp);
  ws->w.sp = e.spill + scratch_slot(e, warp);
  WarpScratch* w = &ws->w;
  join_cta(bs, wsa, w, warp, block_count[blockIdx.x]);
  const MwModel* m = (const MwModel*)bs->model;
  load_env(ws, e.state + env, lane);
  if (lane < 16) w->prof[lane] = 0;
  if (lane == 0) { w->fault = 0; w->prof_on = 0; w->ctrl[0] = actions[4 * env + 3]; w->ctrl[1] = -actions[4 * env + 3]; }
  SYNCW();
  mw_forward(m, e.meshverts[mi], w, lane);
  if (lane == 0) {
    real raw_act[4]; for (int i = 0; i < 4; i++) raw_act[i] = actions[4 * env + i];
    TaskCtx c; c.m = m; c.tc = &bs->tc; c.w = w; c.s = &ws->es; c.action = raw_act; c.meshvert = e.meshverts[mi];
    task_live_update(c);
    real obsr[39]; for (int i = 0; i < 39; i++) obsr[i] = obs_in[(size_t)env * obs_stride + i];
    real rew, inf[INFO_N];
    task_reward(c, obsr, &rew, inf);
    for (int i = 0; i < INFO_N; i++) out[8 * env + i] = (float)inf[i];
    out[8 * env + 7] = (float)rew;
    e.diag[3 * env + 2] |= w->fault;
  }
}

// MujocoEnv.set_state (gymnasium mujoco_env.py) without its mj_forward, one warp per env: envs with mask[env] set take
// qpos[env, :nq] and qvel[env, :nv] of their model (qvel rounded to the record's float32); nothing else of the record
// changes.  The forward pass is not needed: every quantity it derives is recomputed by the next step's first mw_forward
// (or by k_observe), and the only one that outlives a pass, the warm-start qacc, is written by the integrator alone
// (mj_Euler); the stale separating-axis hints can only fail to reject a pair (mw_set_envs)
__global__ void k_set_physics(EngineDev e, const int* __restrict__ env_model, const unsigned char* __restrict__ mask,
                              const double* __restrict__ qpos, const double* __restrict__ qvel) {
  const int env = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (env >= e.n_envs || !mask[env]) return;
  const MwModel* m = (const MwModel*)(e.models + (size_t)env_model[env] * e.model_stride);
  if (lane < m->nq) e.state[env].qpos[lane] = qpos[(size_t)env * MW_MAXNQ + lane];
  if (lane < m->nv) e.state[env].qvel[lane] = (float)qvel[(size_t)env * MW_MAXDOF + lane];
}

// SawyerMocapBase.get_env_state for every env: qpos [n_envs, MW_MAXNQ] float64, qvel [n_envs, MW_MAXDOF] widened to
// float64; columns past the model's nq / nv are zero
__global__ void k_get_physics(EngineDev e, const int* __restrict__ env_model, double* __restrict__ qpos, double* __restrict__ qvel) {
  const int env = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (env >= e.n_envs) return;
  const MwModel* m = (const MwModel*)(e.models + (size_t)env_model[env] * e.model_stride);
  if (lane < MW_MAXNQ) qpos[(size_t)env * MW_MAXNQ + lane] = lane < m->nq ? e.state[env].qpos[lane] : 0.0;
  if (lane < MW_MAXDOF) qvel[(size_t)env * MW_MAXDOF + lane] = lane < m->nv ? (double)e.state[env].qvel[lane] : 0.0;
}

// metaworld.policies' get_action (mw_policies.cuh) for row i of a float32 observation table, one thread per row: the first
// 39 columns widened to double, the policy of task_ids[i], the float32 action.  Reads no engine state
__global__ void k_expert(int n, const int* __restrict__ task_ids, const float* __restrict__ obs, int obs_stride, float* __restrict__ actions) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double o[39];
  const float* row = obs + (size_t)i * obs_stride;
  for (int k = 0; k < 39; k++) o[k] = (double)row[k];
  policy_action(task_ids[i], o, actions + (size_t)i * 4);
}

// SawyerXYZEnv._get_obs (sawyer_xyz_env.py:513-527) of the current state for the envs with mask[env] set: the kinematics
// pass, then the unclipped observation; commits prev_obs (the frame stack) like the reference.  No task's observation
// reads contacts or forces (task_obs_objects: frame poses and qpos only), so the kinematics pass is all of mj_forward
// that it needs.  Barriers: a CTA whose envs are all unmasked leaves before its first barrier (every thread of the CTA
// reads the same mask bytes, so the exit is uniform); in a CTA that stays, the unmasked warps run the same kinematics
// pass as the masked ones and so meet every barrier (the one at the start of mw_forward_kinematics_only), and only
// skip the writes; warps past block_count exit before any barrier and are not counted by it (as in k_step).
__global__ void __launch_bounds__(BLOCK_THREADS, 1)
k_observe(EngineDev e, const int* __restrict__ block_model, const int* __restrict__ block_start, const int* __restrict__ block_count,
          const int* __restrict__ perm, const unsigned char* __restrict__ mask, float* __restrict__ obs_out, int obs_stride) {
  extern __shared__ __align__(16) unsigned char smem[];
  BlockShared* bs = (BlockShared*)smem;
  WarpShared* wsa = (WarpShared*)(smem + sizeof(BlockShared));
  {
    bool any = false;
    for (int k = 0; k < block_count[blockIdx.x]; k++) any = any || mask[perm[block_start[blockIdx.x] + k]];
    if (!any) return;
  }
  const int mi = block_model[blockIdx.x];
  stage_model(bs, e.models + (size_t)mi * e.model_stride, (unsigned)sizeof(bs->model), e.taskconsts + mi);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp >= block_count[blockIdx.x]) return;
  const int env = perm[block_start[blockIdx.x] + warp];
  WarpShared* ws = wsa + warp;
  ws->w.epa = e.epa + scratch_slot(e, warp);
  ws->w.sp = e.spill + scratch_slot(e, warp);
  WarpScratch* w = &ws->w;
  join_cta(bs, wsa, w, warp, block_count[blockIdx.x]);
  const MwModel* m = (const MwModel*)bs->model;
  load_env(ws, e.state + env, lane);
  if (lane < 16) w->prof[lane] = 0;
  if (lane == 0) { w->fault = 0; w->prof_on = 0; }
  SYNCW();
  mw_forward_kinematics_only(m, w, lane);
  if (!mask[env]) return;                              // after the CTA's last barrier
  if (lane == 0) {
    real act[4] = {0, 0, 0, 0};
    TaskCtx c; c.m = m; c.tc = &bs->tc; c.w = w; c.s = &ws->es; c.action = act; c.meshvert = e.meshverts[mi];
    task_live_update(c);                               // _target_pos of the tasks that alias a site (as k_step before make_obs)
    make_obs(c, ws->obs, /*clip=*/false);
    bool fin = true; for (int i = 0; i < 39; i++) fin = fin && isfinite(ws->obs[i]);
    if (!fin) e.diag[3 * env + 2] |= MW_FAULT_NONFINITE;
  }
  SYNCW();
  for (int i = lane; i < 39; i += 32) obs_out[(size_t)env * obs_stride + i] = ws->obs[i];
  ((float4*)(e.state + env))[lane] = ((const float4*)&ws->es)[lane];   // prev_obs (and a live target); the rest as loaded
}

// one named frame of a query table (mw_query; built by metaworld_b200/lower.py query_table): the pose relative to link
// `link`, to the world when link == -1 (translated by the env's shift when MW_QF_SHIFT), or to the mocap body when
// link == MW_QF_MOCAP_LINK
#define MW_QF_SHIFT 1       // a static frame that rides on the task's movable body (model.body(..).pos edits)
#define MW_QF_MISSING 2     // the name does not exist in this model: NaN row
#define MW_QF_TARGET 4      // the position is the env's _target_pos (a site the task keeps aliased to it: basketball's goal)
#define MW_QF_MOCAP_LINK -2 // the frame rides on the mocap body (data.mocap_pos, mocap_quat)
#define MW_QF_ADD_TARGET 8  // a site whose model.site(..).pos reset_model set to _target_pos: + the env's target
#define MW_QF_ADD_OBJ_INIT 16   // the same with obj_init_pos (disassemble's pegTop)
struct MwQueryFrame { int link, flags; double pos[3], quat[4]; };
static_assert(sizeof(MwQueryFrame) == 64, "MwQueryFrame layout mismatch with lower.py QUERY_DTYPE");

// Read-only state query of the envs with mask[env] set (mw_query): the current observation frame (columns 0..17 of the next
// _get_obs, unclipped), world poses of named frames and touching_object of one collider.  Nothing is written back: not the
// record (the frame stack, the live target), the warm start, the separating-axis hints (join_cta without hints) or any fault
// bit but MW_FAULT_NONFINITE.  Barriers as in k_observe: a CTA without a masked env leaves before its first barrier, the
// unmasked warps of a CTA that stays run the same pass and skip the writes, warps past block_count exit before any barrier.
// `touch_geom` non-null: the full forward pass (contacts, constraint forces from the record's gripper command), else the
// kinematics pass only.
__global__ void __launch_bounds__(BLOCK_THREADS, 1)
k_query(EngineDev e, const int* __restrict__ block_model, const int* __restrict__ block_start, const int* __restrict__ block_count,
        const int* __restrict__ perm, const unsigned char* __restrict__ mask, float* __restrict__ frame_out,
        const MwQueryFrame* __restrict__ table, int nq_frames, double* __restrict__ pose_out,
        const int* __restrict__ touch_geom, unsigned char* __restrict__ touching_out) {
  extern __shared__ __align__(16) unsigned char smem[];
  BlockShared* bs = (BlockShared*)smem;
  WarpShared* wsa = (WarpShared*)(smem + sizeof(BlockShared));
  {
    bool any = false;
    for (int k = 0; k < block_count[blockIdx.x]; k++) any = any || mask[perm[block_start[blockIdx.x] + k]];
    if (!any) return;
  }
  const int mi = block_model[blockIdx.x];
  stage_model(bs, e.models + (size_t)mi * e.model_stride, (unsigned)sizeof(bs->model), e.taskconsts + mi);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp >= block_count[blockIdx.x]) return;
  const int env = perm[block_start[blockIdx.x] + warp];
  WarpShared* ws = wsa + warp;
  ws->w.epa = e.epa + scratch_slot(e, warp);
  ws->w.sp = e.spill + scratch_slot(e, warp);
  WarpScratch* w = &ws->w;
  join_cta(bs, wsa, w, warp, block_count[blockIdx.x]);
  const MwModel* m = (const MwModel*)bs->model;
  load_env(ws, e.state + env, lane);
  if (lane < 16) w->prof[lane] = 0;
  if (lane == 0) { w->fault = 0; w->prof_on = 0; w->ctrl[0] = ws->es.gripper_ctrl; w->ctrl[1] = -ws->es.gripper_ctrl; }
  SYNCW();
  if (touching_out) mw_forward(m, e.meshverts[mi], w, lane);
  else mw_forward_kinematics_only(m, w, lane);
  if (!mask[env]) return;                              // after the CTA's last barrier
  real act[4] = {0, 0, 0, 0};
  TaskCtx c; c.m = m; c.tc = &bs->tc; c.w = w; c.s = &ws->es; c.action = act; c.meshvert = e.meshverts[mi];
  if (lane == 0) {
    task_live_update(c);                               // basketball's aliased goal, as before make_obs in k_step
    if (frame_out) {
      make_obs(c, ws->obs, /*clip=*/false);            // also advances ws->es.prev_obs, which is never stored
      bool fin = true; for (int i = 0; i < 18; i++) fin = fin && isfinite(ws->obs[i]);
      if (!fin) e.diag[3 * env + 2] |= MW_FAULT_NONFINITE;
    }
    if (touching_out) { const int g = touch_geom[mi]; touching_out[env] = g >= 0 && touching_object(c, g, (int)bs->tc.p[14], (int)bs->tc.p[15]); }
  }
  SYNCW();
  if (frame_out) for (int i = lane; i < 18; i += 32) frame_out[(size_t)env * 18 + i] = ws->obs[i];
  if (pose_out) {
    for (int k = lane; k < nq_frames; k += 32) {       // one frame per lane, in float64 from the float64 link poses
      const MwQueryFrame f = table[(size_t)mi * nq_frames + k];
      double* o = pose_out + ((size_t)env * nq_frames + k) * 7;
      if (f.flags & MW_QF_MISSING) { for (int i = 0; i < 7; i++) o[i] = __longlong_as_double(0x7ff8000000000000ll); continue; }
      double p[3], q[4];
      if (f.link == -1) {
        for (int i = 0; i < 3; i++) p[i] = f.pos[i] + ((f.flags & MW_QF_SHIFT) ? (double)w->shift[i] : 0.0);
        for (int i = 0; i < 4; i++) q[i] = f.quat[i];
      } else {
        const bool mocap = f.link == MW_QF_MOCAP_LINK;
        double R[9], lq[4], lp[3], t[3];
        for (int i = 0; i < 4; i++) lq[i] = mocap ? (double)w->mocap_quat[i] : w->lquatd[f.link][i];
        for (int i = 0; i < 3; i++) lp[i] = mocap ? (double)w->mocap_pos[i] : w->lposd[f.link][i];
        if (mocap) quat_normalize(lq);
        quat2mat(R, lq); mat_mulvec(t, R, f.pos); v3add(p, lp, t);
        quat_mul(q, lq, f.quat);
      }
      quat_normalize(q);
      if (f.flags & MW_QF_ADD_TARGET) for (int i = 0; i < 3; i++) p[i] += (double)ws->es.target[i];
      if (f.flags & MW_QF_ADD_OBJ_INIT) for (int i = 0; i < 3; i++) p[i] += (double)ws->es.obj_init[i];
      if (f.flags & MW_QF_TARGET) for (int i = 0; i < 3; i++) p[i] = ws->es.target[i];
      for (int i = 0; i < 3; i++) o[i] = p[i];
      for (int i = 0; i < 4; i++) o[3 + i] = q[i];
    }
  }
}

// ---------------------------------------------------------------- launch-order maintenance
// Environments differ several-fold in step cost (contacts, GJK/EPA, solver iterations) and a CTA holds its SM until its
// slowest warp is done.  Cost is strongly correlated from one step to the next, so before every step (a) the envs of each
// model are sorted by their previous cost, which makes CTAs homogeneous, and (b) the CTAs are sorted by the cost of their
// first (= costliest) env, so the hardware's in-order CTA dispatch is longest-processing-time-first.  Pure scheduling:
// results do not depend on the order.
#define MW_SORT_MAX 8192
DEV void bitonic_sort_u64(unsigned long long* k, int P) {
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < P / 2; i += blockDim.x) {
        int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        bool up = (lo & size) == 0;
        unsigned long long a = k[lo], b = k[hi];
        if ((a > b) == up) { k[lo] = b; k[hi] = a; }
      }
    }
  __syncthreads();
}
__global__ void k_order_envs(const int* __restrict__ model_first, const int* __restrict__ model_count, int* __restrict__ perm, const unsigned* __restrict__ env_cost) {
  extern __shared__ unsigned long long keys[];
  const int first = model_first[blockIdx.x], n = model_count[blockIdx.x];
  if (n <= 1 || n > MW_SORT_MAX) return;
  int P = 1; while (P < n) P <<= 1;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    unsigned long long key = ~0ull;
    if (i < n) { int env = perm[first + i]; key = ((unsigned long long)(0xFFFFFFFFu - env_cost[env]) << 32) | (unsigned)env; }
    keys[i] = key;
  }
  bitonic_sort_u64(keys, P);
  // (tried: dealing the heaviest envs one per CTA so that their convex pairs are shared by lighter CTA-mates - the slowest
  //  CTA got 25 % faster, but every CTA of the model then waits for a heavy solver: 3.63 instead of 3.40 ms per step.  Plain
  //  cost order, i.e. CTAs of similar envs, is what is measured fastest.)
  for (int i = threadIdx.x; i < n; i += blockDim.x) perm[first + i] = (int)(keys[i] & 0xFFFFFFFFull);
}
// CTAs in order of decreasing predicted duration (the hardware hands CTAs to SMs in launch order as SMs free up: longest
// first = LPT list scheduling).  Prediction: the longest previous step of the CTA's envs, in cycles of their then-CTAs when
// `env_cycles` is given (a CTA lasts as long as its slowest warp, whatever the reason: contacts, GJK/EPA, model size),
// else the solver-work counter of its first env.
// HEAD SPLIT (opt in, MW_B200_SPLIT_FRAC): k_order_envs keeps a model's envs sorted by cost, so the first CTA of a model holds
// its seven heaviest envs; when those are pathological (a jammed plug, a lid wedged on its box: 5-6 M cycles each against a
// mean of 1.1 M) that one CTA outlasts the balanced load of an SM and IS the duration of the launch.  Fewer resident warps
// run faster each (4 warps: ~1.3 x per warp), so every such model also owns two alternative CTAs that cover the same seven
// envs with `split` and 7 - `split` warps; per step exactly one of {head} / {alt 1, alt 2} is live.  A head is split while its
// predicted duration exceeds `frac` x (sum of the predicted CTA durations / number of SMs), with hysteresis (a split head's
// envs report shorter residences).  Dead CTAs sort last and exit at once.  Pure scheduling: results do not depend on it.
__global__ void k_order_blocks(int n_blocks, const int* __restrict__ block_start, const int* __restrict__ block_count, const int* __restrict__ perm, const unsigned* __restrict__ env_cost,
                               const unsigned* __restrict__ env_cycles, int* __restrict__ block_order,
                               int n_base, int n_split, const int* __restrict__ split_head, const int* __restrict__ split_alt, int* __restrict__ split_state,
                               int* __restrict__ block_live, float frac, int n_sm) {
  extern __shared__ unsigned long long keys[];
  __shared__ unsigned long long total;
  if (n_blocks > MW_SORT_MAX) {
    for (int i = threadIdx.x; i < n_blocks; i += blockDim.x) { block_order[i] = i; if (block_live) block_live[i] = i < n_base; }
    return;
  }
  auto predicted = [&](int i) -> unsigned {
    unsigned c = env_cost[perm[block_start[i]]];
    if (env_cycles) { c = 0; for (int j = 0; j < block_count[i]; j++) c = max(c, env_cycles[perm[block_start[i] + j]]); }
    return c;
  };
  if (block_live) {
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    unsigned long long part = 0;
    for (int i = threadIdx.x; i < n_base; i += blockDim.x) part += predicted(i);
    if (part) atomicAdd(&total, part);
    for (int i = threadIdx.x; i < n_blocks; i += blockDim.x) block_live[i] = i < n_base;
    __syncthreads();
    const float hi = frac * (float)total / (float)(n_sm > 0 ? n_sm : 1), lo = 0.7f * hi;
    for (int s = threadIdx.x; s < n_split; s += blockDim.x) {
      const int h = split_head[s], a1 = split_alt[s];
      const float c = (float)predicted(h);
      int st = split_state[s];
      if (!env_cycles || frac <= 0) st = 0;
      else if (!st && c > hi && hi > 0) st = 1;
      else if (st && c < lo) st = 0;
      split_state[s] = st;
      block_live[h] = !st; block_live[a1] = st; block_live[a1 + 1] = st;
    }
    __syncthreads();
  }
  int P = 1; while (P < n_blocks) P <<= 1;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    unsigned long long key = ~0ull;
    if (i < n_blocks) {
      const unsigned c = (block_live && !block_live[i]) ? 0u : predicted(i);
      key = ((unsigned long long)(0xFFFFFFFFu - c) << 32) | (unsigned)i;
    }
    keys[i] = key;
  }
  bitonic_sort_u64(keys, P);
  for (int i = threadIdx.x; i < n_blocks; i += blockDim.x) block_order[i] = (int)(keys[i] & 0xFFFFFFFFull);
}

// ---------------------------------------------------------------- host side
struct mw_engine {
  int device = 0, n_models = 0, n_envs = 0, model_stride = 0;
  unsigned char* d_models = nullptr; MwTaskConst* d_tc = nullptr; float** d_meshptrs = nullptr;
  std::vector<float*> meshbufs;
  MwEnvState* d_state = nullptr; MwSnapshot* d_snaps = nullptr; int snap_cap = 0, n_snaps = 0;
  int *d_goal_first = nullptr, *d_goal_count = nullptr, *d_diag = nullptr;
  EpaWs* d_epa = nullptr; WarpSpill* d_spill = nullptr; size_t epa_cap = 0; int slot_by_sm = 0, nsmid = 0;
  unsigned long long* d_prof = nullptr; unsigned long long* d_model_cycles = nullptr; unsigned* d_env_prof = nullptr; int profiling = 0;
  float4* d_sep_hint = nullptr;
  unsigned* d_env_cost = nullptr; unsigned* d_env_cycles = nullptr; int order_by_cycles = 1, head_warps = 0; int *d_block_order = nullptr, *d_model_first = nullptr, *d_model_count = nullptr; int n_sorted_models = 0;
  std::vector<int> h_faults;                                   // fault bits already drained from d_diag by mw_get_counters
  std::vector<int> env_model; std::vector<int> model_order;   // block table inputs (mw_rebalance re-sorts the models by measured cost)
  int* d_env_model = nullptr;                                  // env_model on the device (k_set_physics / k_get_physics read each env's nq / nv)
  // env block table
  int n_blocks = 0; int *d_block_model = nullptr, *d_block_start = nullptr, *d_block_count = nullptr, *d_perm = nullptr;
  // head split (k_order_blocks): the alternative CTAs follow the n_blocks regular ones in the block table
  int n_blocks_total = 0, n_split = 0, split_warps = 4, n_sm = 0; float split_frac = 0.f;
  int *d_split_head = nullptr, *d_split_alt = nullptr, *d_split_state = nullptr, *d_block_live = nullptr;
  int max_steps = 500, terminate_on_success = 0; unsigned long long seed = 0; int autoreset_mode = MW_AUTORESET_SAME_STEP;
  unsigned long long launches = 0, env_steps = 0;
  EngineDev dev() const {
    EngineDev e; e.models = d_models; e.model_stride = model_stride; e.taskconsts = d_tc; e.meshverts = d_meshptrs;
    e.state = d_state; e.snaps = d_snaps; e.goal_first = d_goal_first; e.goal_count = d_goal_count; e.diag = d_diag; e.epa = d_epa; e.spill = d_spill; e.slot_by_sm = slot_by_sm; e.prof = profiling ? d_prof : nullptr; e.model_cycles = d_model_cycles; e.env_cost = d_env_cost; e.env_cycles = order_by_cycles ? d_env_cycles : nullptr; e.env_prof = profiling ? d_env_prof : nullptr;
    e.sep_hint = d_sep_hint;
    e.n_envs = n_envs; e.max_steps = max_steps; e.terminate_on_success = terminate_on_success; e.seed = seed; e.autoreset_mode = autoreset_mode; return e;
  }
};

// group work items by model into CTAs of WARPS_PER_BLOCK warps
// `order` (optional): models in launch order -- the costliest first, so that the hardware's in-order CTA dispatch behaves
// like longest-processing-time-first list scheduling and the cheap CTAs fill the tail
// `head`: size of the FIRST CTA of every model (0 = full; the partial CTA of a model is then its last).  k_order_envs keeps
// a model's envs sorted by cost, so the first CTA holds its heaviest envs, and with fewer resident warps each of them
// runs faster (5 warps: ~1.2x per warp).  Measured (MW_B200_HEAD_WARPS, MT50 @ 4096 steady state): 3.42 ms with head 0,
// 3.46 with the partial CTA first (-1 -> count % WARPS_PER_BLOCK), 3.58 / 3.63 / 3.64 with heads of 4 / 3 / 2 -- the SM
// that hosts a small CTA is under-used for that CTA's whole life, and in steady state the mean load, not the slowest
// env, bounds the launch.  Kept as a switch for that measurement only.
static void make_blocks(int n_models, const std::vector<int>& item_model, std::vector<int>& bm, std::vector<int>& bstart, std::vector<int>& bcount, std::vector<int>& perm,
                        const std::vector<int>* order = nullptr, int head = 0) {
  bm.clear(); bstart.clear(); bcount.clear(); perm.clear();
  for (int oi = 0; oi < n_models; oi++) {
    const int mi = order && (int)order->size() == n_models ? (*order)[oi] : oi;
    int first = (int)perm.size();
    for (int i = 0; i < (int)item_model.size(); i++) if (item_model[i] == mi) perm.push_back(i);
    int cnt = (int)perm.size() - first;
    int h = head < 0 ? cnt % WARPS_PER_BLOCK : head;
    if (h <= 0 || h > WARPS_PER_BLOCK) h = WARPS_PER_BLOCK;
    for (int o = 0; o < cnt; ) {
      const int take = std::min(o == 0 ? h : WARPS_PER_BLOCK, cnt - o);
      bm.push_back(mi); bstart.push_back(first + o); bcount.push_back(take);
      o += take;
    }
  }
}
static int ensure_epa(mw_engine* E, size_t n_blocks) {
  if (E->nsmid == 0) {
    // one CTA per SM whenever two CTAs' shared memory cannot fit (true for every build so far: 190-227 KB per CTA)
    int dev = 0; cudaDeviceProp pr; CK(cudaGetDevice(&dev)); CK(cudaGetDeviceProperties(&pr, dev));
    unsigned* d_n = nullptr; unsigned h_n = 0;
    CK(cudaMalloc((void**)&d_n, sizeof(unsigned)));
    k_nsmid<<<1, 1>>>(d_n);
    CK(cudaMemcpy(&h_n, d_n, sizeof(unsigned), cudaMemcpyDeviceToHost)); cudaFree(d_n);
    E->nsmid = (int)h_n;
    E->slot_by_sm = (2 * smem_bytes() > (size_t)pr.sharedMemPerMultiprocessor && h_n > 0 && h_n <= 4096) ? 1 : 0;
  }
  size_t need = (E->slot_by_sm ? (size_t)E->nsmid : n_blocks) * WARPS_PER_BLOCK;
  if (need <= E->epa_cap) return 0;
  if (E->d_epa) cudaFree(E->d_epa);
  if (E->d_spill) cudaFree(E->d_spill);
  E->d_epa = nullptr; E->d_spill = nullptr; E->epa_cap = 0;
  CK(cudaMalloc((void**)&E->d_epa, sizeof(EpaWs) * need));
  CK(cudaMalloc((void**)&E->d_spill, sizeof(WarpSpill) * need));
  E->epa_cap = need;
  return 0;
}
template <class T> static int upload(T** dst, const std::vector<T>& v) {
  if (*dst) cudaFree(*dst);
  *dst = nullptr;
  CK(cudaMalloc((void**)dst, sizeof(T) * (v.size() ? v.size() : 1)));
  if (!v.empty()) CK(cudaMemcpy(*dst, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
  return 0;
}

// (re)builds and uploads the CTA table of the environment set + the buffers of the launch-order kernels
static int upload_env_blocks(mw_engine* E) {
  std::vector<int> bm, bs, bc, perm;
  make_blocks(E->n_models, E->env_model, bm, bs, bc, perm, &E->model_order, E->head_warps);
  E->n_blocks = (int)bm.size();
  std::vector<int> mfirst, mcount;
  for (size_t b = 0; b < bm.size(); b++) {
    if (b == 0 || bm[b] != bm[b - 1]) { mfirst.push_back(bs[b]); mcount.push_back(0); }
    mcount.back() += bc[b];
  }
  // alternative decomposition of every full first CTA of a model (head split, see k_order_blocks)
  std::vector<int> shead, salt;
  const int sw = E->split_warps;
  if (E->split_frac > 0 && sw > 0 && sw < WARPS_PER_BLOCK) {
    const size_t nb = bm.size();
    for (size_t b = 0; b < nb; b++) {
      if ((b == 0 || bm[b] != bm[b - 1]) && bc[b] == WARPS_PER_BLOCK) {
        shead.push_back((int)b); salt.push_back((int)bm.size());
        bm.push_back(bm[b]); bs.push_back(bs[b]); bc.push_back(sw);
        bm.push_back(bm[b]); bs.push_back(bs[b] + sw); bc.push_back(WARPS_PER_BLOCK - sw);
      }
    }
  }
  E->n_split = (int)shead.size(); E->n_blocks_total = (int)bm.size();
  if (ensure_epa(E, bm.size())) return MW_ERR_CUDA;
  if (upload(&E->d_block_model, bm) || upload(&E->d_block_start, bs) || upload(&E->d_block_count, bc) || upload(&E->d_perm, perm)) return MW_ERR_CUDA;
  std::vector<int> order(bm.size()), live(bm.size()), zero(shead.size() ? shead.size() : 1, 0);
  for (size_t b = 0; b < bm.size(); b++) { order[b] = (int)b; live[b] = b < (size_t)E->n_blocks; }
  E->n_sorted_models = (int)mfirst.size();
  if (upload(&E->d_model_first, mfirst) || upload(&E->d_model_count, mcount) || upload(&E->d_block_order, order)) return MW_ERR_CUDA;
  if (upload(&E->d_split_head, shead) || upload(&E->d_split_alt, salt) || upload(&E->d_split_state, zero) || upload(&E->d_block_live, live)) return MW_ERR_CUDA;
  return 0;
}

extern "C" {

int mw_sizeof_model(void) { return (int)sizeof(MwModel); }
int mw_sizeof_taskconst(void) { return (int)sizeof(MwTaskConst); }
int mw_sizeof_envstate(void) { return (int)sizeof(MwEnvState); }
int mw_sizeof_snapshot(void) { return (int)sizeof(MwSnapshot); }
const char* mw_last_error(void) { return g_err.c_str(); }
const char* mw_build_info(void) {
  static char buf[256];
  snprintf(buf, sizeof(buf), "real=%s maxcon=%d(shared %d) maxefc=%d(shared %d) warps_per_block=%d smem_per_block=%zu", sizeof(real) == 4 ? "float" : "double",
           MW_MAXCON, MW_SMCON, MW_MAXEFC, MW_SMEFC, WARPS_PER_BLOCK, smem_bytes());
  return buf;
}

int mw_create(mw_engine** out, int device, int n_models, const void* models, const void* taskconsts, const float* const* meshverts, const int* nmeshvert) {
  if (!out || n_models <= 0 || !models || !taskconsts) return fail(MW_ERR_ARG, "mw_create: bad arguments");
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(MW_ERR_CUDA, "mw_create: no such CUDA device (this engine has no CPU path)");
  CK(cudaSetDevice(device));
  mw_engine* E = new mw_engine();
  E->device = device; E->n_models = n_models;
  E->model_stride = (int)((sizeof(MwModel) + 15) / 16 * 16);
  std::vector<unsigned char> blob((size_t)E->model_stride * n_models, 0);
  for (int i = 0; i < n_models; i++) memcpy(blob.data() + (size_t)i * E->model_stride, (const unsigned char*)models + (size_t)i * sizeof(MwModel), sizeof(MwModel));
  CK(cudaMalloc((void**)&E->d_models, blob.size()));
  CK(cudaMemcpy(E->d_models, blob.data(), blob.size(), cudaMemcpyHostToDevice));
  CK(cudaMalloc((void**)&E->d_tc, sizeof(MwTaskConst) * n_models));
  CK(cudaMemcpy(E->d_tc, taskconsts, sizeof(MwTaskConst) * n_models, cudaMemcpyHostToDevice));
  std::vector<float*> ptrs(n_models, nullptr);
  for (int i = 0; i < n_models; i++) {
    int nvt = nmeshvert ? nmeshvert[i] : 0;
    float* p = nullptr;
    CK(cudaMalloc((void**)&p, sizeof(float) * 4 * (nvt > 0 ? nvt : 1)));
    if (nvt > 0) {   // repack xyz -> xyz_ so that a support query reads one 16-byte word per vertex
      std::vector<float> packed(4 * (size_t)nvt, 0.f);
      for (int v = 0; v < nvt; v++) for (int c = 0; c < 3; c++) packed[4 * v + c] = meshverts[i][3 * v + c];
      CK(cudaMemcpy(p, packed.data(), sizeof(float) * 4 * nvt, cudaMemcpyHostToDevice));
    }
    ptrs[i] = p; E->meshbufs.push_back(p);
  }
  CK(cudaMalloc((void**)&E->d_meshptrs, sizeof(float*) * n_models));
  CK(cudaMemcpy(E->d_meshptrs, ptrs.data(), sizeof(float*) * n_models, cudaMemcpyHostToDevice));
  CK(cudaMalloc((void**)&E->d_model_cycles, sizeof(unsigned long long) * 2 * n_models));
  CK(cudaMemset(E->d_model_cycles, 0, sizeof(unsigned long long) * 2 * n_models));
  CK(cudaMalloc((void**)&E->d_prof, sizeof(unsigned long long) * 16));
  CK(cudaMemset(E->d_prof, 0, sizeof(unsigned long long) * 16));
  CK(cudaFuncSetAttribute(k_order_envs, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(unsigned long long) * MW_SORT_MAX)));
  CK(cudaFuncSetAttribute(k_order_blocks, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(unsigned long long) * MW_SORT_MAX)));
  CK(cudaFuncSetAttribute(k_step<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
  CK(cudaFuncSetAttribute(k_step<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
  CK(cudaFuncSetAttribute(k_snapshot, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
  CK(cudaFuncSetAttribute(k_substeps, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
  CK(cudaFuncSetAttribute(k_evaluate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
  CK(cudaFuncSetAttribute(k_observe, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
  CK(cudaFuncSetAttribute(k_query, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
  { const char* k = getenv("MW_B200_ORDER_KEY"); if (k && !strcmp(k, "work")) E->order_by_cycles = 0; }   // A/B switches of the launch order
  { const char* k = getenv("MW_B200_HEAD_WARPS"); if (k) E->head_warps = atoi(k); }
  { const char* k = getenv("MW_B200_SPLIT_FRAC"); if (k) E->split_frac = (float)atof(k); }
  { const char* k = getenv("MW_B200_SPLIT_WARPS"); if (k) E->split_warps = atoi(k); }
  { cudaDeviceProp pr; CK(cudaGetDeviceProperties(&pr, device)); E->n_sm = pr.multiProcessorCount; }
  *out = E;
  return MW_OK;
}

void mw_destroy(mw_engine* E) {
  if (!E) return;
  cudaSetDevice(E->device);
  cudaFree(E->d_models); cudaFree(E->d_tc); cudaFree(E->d_meshptrs);
  for (float* p : E->meshbufs) cudaFree(p);
  cudaFree(E->d_state); cudaFree(E->d_snaps); cudaFree(E->d_goal_first); cudaFree(E->d_goal_count); cudaFree(E->d_diag); cudaFree(E->d_epa); cudaFree(E->d_spill); cudaFree(E->d_prof); cudaFree(E->d_model_cycles); cudaFree(E->d_env_prof); cudaFree(E->d_env_cost); cudaFree(E->d_env_cycles); cudaFree(E->d_sep_hint); cudaFree(E->d_env_model); cudaFree(E->d_block_order); cudaFree(E->d_model_first); cudaFree(E->d_model_count);
  cudaFree(E->d_block_model); cudaFree(E->d_block_start); cudaFree(E->d_block_count); cudaFree(E->d_perm);
  cudaFree(E->d_split_head); cudaFree(E->d_split_alt); cudaFree(E->d_split_state); cudaFree(E->d_block_live);
  delete E;
}

int mw_set_envs(mw_engine* E, int n_envs, const int* env_model) {
  if (!E || n_envs <= 0 || !env_model) return fail(MW_ERR_ARG, "mw_set_envs: bad arguments");
  CK(cudaSetDevice(E->device));
  std::vector<int> im(env_model, env_model + n_envs), bm, bs, bc, perm;
  for (int v : im) if (v < 0 || v >= E->n_models) return fail(MW_ERR_ARG, "mw_set_envs: model index out of range");
  E->env_model = im;
  E->n_envs = n_envs;
  E->h_faults.assign(n_envs, 0);
  if (upload_env_blocks(E) || upload(&E->d_env_model, im)) return MW_ERR_CUDA;
  if (E->d_env_cost) cudaFree(E->d_env_cost);
  CK(cudaMalloc((void**)&E->d_env_cost, sizeof(unsigned) * n_envs));
  CK(cudaMemset(E->d_env_cost, 0, sizeof(unsigned) * n_envs));
  if (E->d_env_cycles) cudaFree(E->d_env_cycles);
  CK(cudaMalloc((void**)&E->d_env_cycles, sizeof(unsigned) * n_envs));
  CK(cudaMemset(E->d_env_cycles, 0, sizeof(unsigned) * n_envs));
  // zeroed = no hint anywhere.  Never invalidated: a stale hint can only fail to reject a pair (sep_hint_test), so resets,
  // set_state and checkpoints leave the table alone
  if (E->d_sep_hint) cudaFree(E->d_sep_hint);
  CK(cudaMalloc((void**)&E->d_sep_hint, sizeof(float4) * MW_NCONV * n_envs));
  CK(cudaMemset(E->d_sep_hint, 0, sizeof(float4) * MW_NCONV * n_envs));
  if (E->d_state) cudaFree(E->d_state);
  CK(cudaMalloc((void**)&E->d_state, sizeof(MwEnvState) * n_envs));
  CK(cudaMemset(E->d_state, 0, sizeof(MwEnvState) * n_envs));
  if (E->d_env_prof) { cudaFree(E->d_env_prof); E->d_env_prof = nullptr; }
  if (E->profiling) { CK(cudaMalloc((void**)&E->d_env_prof, sizeof(unsigned) * MW_ENVPROF_W * n_envs)); CK(cudaMemset(E->d_env_prof, 0, sizeof(unsigned) * MW_ENVPROF_W * n_envs)); }
  if (E->d_diag) cudaFree(E->d_diag);
  CK(cudaMalloc((void**)&E->d_diag, sizeof(int) * 3 * n_envs));
  CK(cudaMemset(E->d_diag, 0, sizeof(int) * 3 * n_envs));
  return MW_OK;
}

int mw_build_snapshots(mw_engine* E, int n, const int* model_idx, const double* rand_vec, const double* rand_vec_pass1, const unsigned char* partial, int* ids_out) {
  if (!E || n <= 0 || !model_idx || !rand_vec || !partial) return fail(MW_ERR_ARG, "mw_build_snapshots: bad arguments");
  CK(cudaSetDevice(E->device));
  if (E->n_snaps + n > E->snap_cap) {
    int cap = (E->n_snaps + n) * 2;
    MwSnapshot* p = nullptr;
    CK(cudaMalloc((void**)&p, sizeof(MwSnapshot) * cap));
    if (E->n_snaps) CK(cudaMemcpy(p, E->d_snaps, sizeof(MwSnapshot) * E->n_snaps, cudaMemcpyDeviceToDevice));
    cudaFree(E->d_snaps); E->d_snaps = p; E->snap_cap = cap;
  }
  std::vector<int> im(model_idx, model_idx + n), bm, bs, bc, perm;
  for (int v : im) if (v < 0 || v >= E->n_models) return fail(MW_ERR_ARG, "mw_build_snapshots: model index out of range");
  make_blocks(E->n_models, im, bm, bs, bc, perm);
  if (ensure_epa(E, bm.size())) return MW_ERR_CUDA;
  int *d_bm = nullptr, *d_bs = nullptr, *d_bc = nullptr, *d_perm = nullptr; double* d_rv = nullptr; unsigned char* d_po = nullptr;
  if (upload(&d_bm, bm) || upload(&d_bs, bs) || upload(&d_bc, bc) || upload(&d_perm, perm)) return MW_ERR_CUDA;
  CK(cudaMalloc((void**)&d_rv, sizeof(double) * 6 * n)); CK(cudaMemcpy(d_rv, rand_vec, sizeof(double) * 6 * n, cudaMemcpyHostToDevice));
  CK(cudaMalloc((void**)&d_po, n)); CK(cudaMemcpy(d_po, partial, n, cudaMemcpyHostToDevice));
  double* d_rv1 = nullptr;
  if (rand_vec_pass1) { CK(cudaMalloc((void**)&d_rv1, sizeof(double) * 6 * n)); CK(cudaMemcpy(d_rv1, rand_vec_pass1, sizeof(double) * 6 * n, cudaMemcpyHostToDevice)); }
  k_snapshot<<<(int)bm.size(), BLOCK_THREADS, smem_bytes()>>>(E->dev(), d_bm, d_bs, d_bc, d_perm, d_rv, d_rv1, d_po, E->n_snaps);
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  cudaFree(d_bm); cudaFree(d_bs); cudaFree(d_bc); cudaFree(d_perm); cudaFree(d_rv); cudaFree(d_rv1); cudaFree(d_po);
  if (ids_out) for (int i = 0; i < n; i++) ids_out[i] = E->n_snaps + i;
  E->n_snaps += n; E->launches++;
  return MW_OK;
}
int mw_append_snapshots(mw_engine* E, int n, const void* records, int* ids_out) {
  if (!E || n <= 0 || !records) return fail(MW_ERR_ARG, "mw_append_snapshots: bad arguments");
  CK(cudaSetDevice(E->device));
  if (E->n_snaps + n > E->snap_cap) {
    int cap = (E->n_snaps + n) * 2;
    MwSnapshot* p = nullptr;
    CK(cudaMalloc((void**)&p, sizeof(MwSnapshot) * cap));
    if (E->n_snaps) CK(cudaMemcpy(p, E->d_snaps, sizeof(MwSnapshot) * E->n_snaps, cudaMemcpyDeviceToDevice));
    cudaFree(E->d_snaps); E->d_snaps = p; E->snap_cap = cap;
  }
  std::vector<MwSnapshot> tmp((const MwSnapshot*)records, (const MwSnapshot*)records + n);
  for (int i = 0; i < n; i++) tmp[i].st.snapshot = (float)(E->n_snaps + i);
  CK(cudaMemcpy(E->d_snaps + E->n_snaps, tmp.data(), sizeof(MwSnapshot) * n, cudaMemcpyHostToDevice));
  if (ids_out) for (int i = 0; i < n; i++) ids_out[i] = E->n_snaps + i;
  E->n_snaps += n;
  return MW_OK;
}
int mw_num_snapshots(const mw_engine* E) { return E ? E->n_snaps : 0; }
int mw_get_snapshots(mw_engine* E, int first, int n, void* out) {
  if (!E || first < 0 || first + n > E->n_snaps) return fail(MW_ERR_ARG, "mw_get_snapshots: range");
  CK(cudaSetDevice(E->device));
  CK(cudaMemcpy(out, E->d_snaps + first, sizeof(MwSnapshot) * n, cudaMemcpyDeviceToHost));
  return MW_OK;
}

int mw_reset(mw_engine* E, int n, const int* env_ids, const int* snapshot_ids, float* obs, int obs_stride, void* stream) {
  if (!E || !E->d_state || n <= 0 || !snapshot_ids || !obs || obs_stride < 39) return fail(MW_ERR_ARG, "mw_reset: bad arguments");
  CK(cudaSetDevice(E->device));
  k_reset<<<(n * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(E->dev(), n, env_ids, snapshot_ids, obs, obs_stride);
  CK(cudaGetLastError());
  E->launches++;
  return MW_OK;
}

int mw_reset_masked(mw_engine* E, const unsigned char* mask, const int* snapshot_ids, float* obs, int obs_stride, void* stream) {
  if (!E || !E->d_state) return fail(MW_ERR_STATE, "mw_reset_masked: mw_set_envs not called");
  if (!mask || !obs || obs_stride < 39) return fail(MW_ERR_ARG, "mw_reset_masked: bad arguments");
  if (!snapshot_ids && !E->d_goal_first) return fail(MW_ERR_STATE, "mw_reset_masked: no snapshot_ids and no goal sets for the device sampler");
  CK(cudaSetDevice(E->device));
  k_reset_masked<<<(E->n_envs * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(E->dev(), mask, snapshot_ids, obs, obs_stride);
  CK(cudaGetLastError());
  E->launches++;
  return MW_OK;
}

int mw_set_autoreset_mode(mw_engine* E, int mode) {
  if (!E || (mode != MW_AUTORESET_SAME_STEP && mode != MW_AUTORESET_NEXT_STEP && mode != MW_AUTORESET_DISABLED))
    return fail(MW_ERR_ARG, "mw_set_autoreset_mode: mode must be MW_AUTORESET_SAME_STEP, _NEXT_STEP or _DISABLED");
  E->autoreset_mode = mode;
  return MW_OK;
}

int mw_step(mw_engine* E, const float* actions, float* obs, int obs_stride, float* reward, unsigned char* terminated, unsigned char* truncated,
            float* info, int info_stride, float* final_obs, float* final_info, const int* next_snapshot, void* stream) {
  if (!E || !E->d_state) return fail(MW_ERR_STATE, "mw_step: mw_set_envs not called");
  if (!actions || !obs || !reward || !terminated || !truncated || !info || obs_stride < 39 || info_stride < 7) return fail(MW_ERR_ARG, "mw_step: bad arguments");
  if (!next_snapshot && !E->d_goal_first) return fail(MW_ERR_STATE, "mw_step: no next_snapshot and no goal sets for the device sampler");
  CK(cudaSetDevice(E->device));
  {   // launch order from the previous step's per-env cost (see k_order_*)
    int Pm = 1; while (Pm < E->n_envs && Pm < MW_SORT_MAX) Pm <<= 1;
    const int nb = E->n_split ? E->n_blocks_total : E->n_blocks;
    int Pb = 1; while (Pb < nb && Pb < MW_SORT_MAX) Pb <<= 1;
    k_order_envs<<<E->n_sorted_models, 1024, sizeof(unsigned long long) * Pm, (cudaStream_t)stream>>>(E->d_model_first, E->d_model_count, E->d_perm, E->d_env_cost);
    k_order_blocks<<<1, 1024, sizeof(unsigned long long) * Pb, (cudaStream_t)stream>>>(nb, E->d_block_start, E->d_block_count, E->d_perm, E->d_env_cost, E->order_by_cycles ? E->d_env_cycles : nullptr, E->d_block_order,
        E->n_blocks, E->n_split, E->d_split_head, E->d_split_alt, E->d_split_state, E->n_split ? E->d_block_live : nullptr, E->split_frac, E->n_sm);
  }
  auto* kern = E->autoreset_mode == MW_AUTORESET_SAME_STEP ? k_step<false> : k_step<true>;
  kern<<<E->n_split ? E->n_blocks_total : E->n_blocks, BLOCK_THREADS, smem_bytes(), (cudaStream_t)stream>>>(E->dev(), E->d_block_order, E->d_block_model, E->d_block_start, E->d_block_count, E->d_perm,
      actions, obs, obs_stride, reward, terminated, truncated, info, info_stride, final_obs, final_info, next_snapshot, E->n_split ? E->d_block_live : nullptr);
  CK(cudaGetLastError());
  E->launches += 3; E->env_steps += (unsigned long long)E->n_envs;
  return MW_OK;
}

int mw_evaluate(mw_engine* E, const float* actions, const float* obs, int obs_stride, float* out, void* stream) {
  if (!E || !E->d_state || !actions || !obs || !out || obs_stride < 39) return fail(MW_ERR_ARG, "mw_evaluate: bad arguments");
  CK(cudaSetDevice(E->device));
  k_evaluate<<<E->n_blocks, BLOCK_THREADS, smem_bytes(), (cudaStream_t)stream>>>(E->dev(), E->d_block_model, E->d_block_start, E->d_block_count, E->d_perm, actions, obs, obs_stride, out);
  CK(cudaGetLastError());
  E->launches++;
  return MW_OK;
}

int mw_set_physics(mw_engine* E, const unsigned char* mask, const double* qpos, const double* qvel, void* stream) {
  if (!E || !E->d_state) return fail(MW_ERR_STATE, "mw_set_physics: mw_set_envs not called");
  if (!mask || !qpos || !qvel) return fail(MW_ERR_ARG, "mw_set_physics: bad arguments");
  CK(cudaSetDevice(E->device));
  k_set_physics<<<(E->n_envs * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(E->dev(), E->d_env_model, mask, qpos, qvel);
  CK(cudaGetLastError());
  E->launches++;
  return MW_OK;
}

int mw_get_physics(mw_engine* E, double* qpos, double* qvel, void* stream) {
  if (!E || !E->d_state) return fail(MW_ERR_STATE, "mw_get_physics: mw_set_envs not called");
  if (!qpos || !qvel) return fail(MW_ERR_ARG, "mw_get_physics: bad arguments");
  CK(cudaSetDevice(E->device));
  k_get_physics<<<(E->n_envs * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(E->dev(), E->d_env_model, qpos, qvel);
  CK(cudaGetLastError());
  E->launches++;
  return MW_OK;
}

int mw_observe(mw_engine* E, const unsigned char* mask, float* obs, int obs_stride, void* stream) {
  if (!E || !E->d_state) return fail(MW_ERR_STATE, "mw_observe: mw_set_envs not called");
  if (!mask || !obs || obs_stride < 39) return fail(MW_ERR_ARG, "mw_observe: bad arguments");
  CK(cudaSetDevice(E->device));
  k_observe<<<E->n_blocks, BLOCK_THREADS, smem_bytes(), (cudaStream_t)stream>>>(E->dev(), E->d_block_model, E->d_block_start, E->d_block_count, E->d_perm, mask, obs, obs_stride);
  CK(cudaGetLastError());
  E->launches++;
  return MW_OK;
}

int mw_query(mw_engine* E, const unsigned char* mask, float* frame, const void* frames, int n_frames, double* pose,
             const int* touch_geom, unsigned char* touching, void* stream) {
  if (!E || !E->d_state) return fail(MW_ERR_STATE, "mw_query: mw_set_envs not called");
  if (!mask || n_frames < 0 || (pose && (!frames || n_frames == 0)) || (!touching) != (!touch_geom))
    return fail(MW_ERR_ARG, "mw_query: bad arguments");
  if (!frame && !pose && !touching) return MW_OK;
  CK(cudaSetDevice(E->device));
  k_query<<<E->n_blocks, BLOCK_THREADS, smem_bytes(), (cudaStream_t)stream>>>(E->dev(), E->d_block_model, E->d_block_start, E->d_block_count, E->d_perm,
      mask, frame, (const MwQueryFrame*)frames, pose ? n_frames : 0, pose, touch_geom, touching);
  CK(cudaGetLastError());
  E->launches++;
  return MW_OK;
}

int mw_expert_actions(const int* task_ids, const float* obs, int obs_stride, int n, float* actions, void* stream) {
  if (n < 0 || obs_stride < 39 || (n > 0 && (!task_ids || !obs || !actions))) return fail(MW_ERR_ARG, "mw_expert_actions: bad arguments");
  if (n == 0) return MW_OK;
  k_expert<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n, task_ids, obs, obs_stride, actions);
  CK(cudaGetLastError());
  return MW_OK;
}

int mw_get_faults(mw_engine* E, int* out) {
  if (!E || !out || !E->d_diag) return fail(MW_ERR_ARG, "mw_get_faults");
  CK(cudaSetDevice(E->device));
  std::vector<int> diag(3 * (size_t)E->n_envs);
  CK(cudaMemcpy(diag.data(), E->d_diag, sizeof(int) * diag.size(), cudaMemcpyDeviceToHost));
  for (int i = 0; i < E->n_envs; i++) { out[i] = E->h_faults[i] | diag[3 * i + 2]; E->h_faults[i] = 0; diag[3 * i + 2] = 0; }
  CK(cudaMemcpy(E->d_diag, diag.data(), sizeof(int) * diag.size(), cudaMemcpyHostToDevice));
  return MW_OK;
}

int mw_set_options(mw_engine* E, int max_episode_steps, int terminate_on_success, unsigned long long seed) {
  if (!E || max_episode_steps <= 0) return fail(MW_ERR_ARG, "mw_set_options: bad arguments");
  E->max_steps = max_episode_steps; E->terminate_on_success = terminate_on_success; E->seed = seed;
  return MW_OK;
}
int mw_set_goal_sets(mw_engine* E, const int* first, const int* count) {
  if (!E || !E->n_envs || !first || !count) return fail(MW_ERR_ARG, "mw_set_goal_sets: bad arguments");
  CK(cudaSetDevice(E->device));
  std::vector<int> f(first, first + E->n_envs), c(count, count + E->n_envs);
  for (int i = 0; i < E->n_envs; i++) if (c[i] <= 0 || f[i] < 0 || f[i] + c[i] > E->n_snaps) return fail(MW_ERR_ARG, "mw_set_goal_sets: range outside the snapshot table");
  if (upload(&E->d_goal_first, f) || upload(&E->d_goal_count, c)) return MW_ERR_CUDA;
  return MW_OK;
}
int mw_get_state(mw_engine* E, void* out) {
  if (!E || !E->d_state || !out) return fail(MW_ERR_ARG, "mw_get_state");
  CK(cudaSetDevice(E->device));
  CK(cudaMemcpy(out, E->d_state, sizeof(MwEnvState) * E->n_envs, cudaMemcpyDeviceToHost));
  return MW_OK;
}
int mw_set_state(mw_engine* E, const void* in) {
  if (!E || !E->d_state || !in) return fail(MW_ERR_ARG, "mw_set_state");
  CK(cudaSetDevice(E->device));
  CK(cudaMemcpy(E->d_state, in, sizeof(MwEnvState) * E->n_envs, cudaMemcpyHostToDevice));
  return MW_OK;
}
int mw_debug_substeps(mw_engine* E, int nstep, const float* ctrl2, void* stream) {
  if (!E || !E->d_state || nstep < 0 || !ctrl2) return fail(MW_ERR_ARG, "mw_debug_substeps");
  CK(cudaSetDevice(E->device));
  k_substeps<<<E->n_blocks, BLOCK_THREADS, smem_bytes(), (cudaStream_t)stream>>>(E->dev(), E->d_block_model, E->d_block_start, E->d_block_count, E->d_perm, nstep, ctrl2[0], ctrl2[1], nullptr);
  CK(cudaGetLastError());
  E->launches++;
  return MW_OK;
}
int mw_debug_forward(mw_engine* E, const float* ctrl2, float* dump_dev, void* stream) {
  if (!E || !E->d_state || !ctrl2 || !dump_dev) return fail(MW_ERR_ARG, "mw_debug_forward");
  CK(cudaSetDevice(E->device));
  k_substeps<<<E->n_blocks, BLOCK_THREADS, smem_bytes(), (cudaStream_t)stream>>>(E->dev(), E->d_block_model, E->d_block_start, E->d_block_count, E->d_perm, 0, ctrl2[0], ctrl2[1], dump_dev);
  CK(cudaGetLastError());
  return MW_OK;
}
int mw_debug_dump_floats(void) { return MW_MAXCON * 12 + MW_MAXDOF + 4; }
int mw_get_counters(mw_engine* E, unsigned long long* out5) {
  if (!E || !out5) return fail(MW_ERR_ARG, "mw_get_counters");
  CK(cudaSetDevice(E->device));
  std::vector<int> diag(3 * (size_t)(E->n_envs > 0 ? E->n_envs : 0));
  if (E->n_envs) {
    CK(cudaMemcpy(diag.data(), E->d_diag, sizeof(int) * diag.size(), cudaMemcpyDeviceToHost));
    for (int i = 0; i < E->n_envs; i++) { E->h_faults[i] |= diag[3 * i + 2]; }
    CK(cudaMemset(E->d_diag, 0, sizeof(int) * diag.size()));
  }
  unsigned long long dropped = 0, iters = 0;
  for (int i = 0; i < E->n_envs; i++) { dropped += diag[3 * i]; iters += diag[3 * i + 1]; }
  out5[0] = E->launches; out5[1] = E->env_steps; out5[2] = dropped; out5[3] = iters; out5[4] = E->env_steps * 6ull;
  E->launches = 0; E->env_steps = 0;
  return MW_OK;
}

int mw_rebalance(mw_engine* E) {
  if (!E || !E->d_state) return fail(MW_ERR_STATE, "mw_rebalance: mw_set_envs not called");
  CK(cudaSetDevice(E->device));
  CK(cudaDeviceSynchronize());
  std::vector<unsigned long long> mc(2 * (size_t)E->n_models);
  CK(cudaMemcpy(mc.data(), E->d_model_cycles, sizeof(unsigned long long) * mc.size(), cudaMemcpyDeviceToHost));
  CK(cudaMemset(E->d_model_cycles, 0, sizeof(unsigned long long) * mc.size()));
  std::vector<std::pair<double, int>> cost;
  for (int i = 0; i < E->n_models; i++) cost.push_back({mc[2 * i + 1] ? (double)mc[2 * i] / (double)mc[2 * i + 1] : 0.0, i});
  std::stable_sort(cost.begin(), cost.end(), [](const std::pair<double, int>& a, const std::pair<double, int>& b) { return a.first > b.first; });
  E->model_order.clear();
  for (auto& c : cost) E->model_order.push_back(c.second);
  if (upload_env_blocks(E)) return MW_ERR_CUDA;
  return MW_OK;
}

int mw_set_profiling(mw_engine* E, int on) {
  if (!E) return fail(MW_ERR_ARG, "mw_set_profiling");
  CK(cudaSetDevice(E->device));
  E->profiling = on ? 1 : 0;
  if (on && E->n_envs && !E->d_env_prof) { CK(cudaMalloc((void**)&E->d_env_prof, sizeof(unsigned) * MW_ENVPROF_W * E->n_envs)); CK(cudaMemset(E->d_env_prof, 0, sizeof(unsigned) * MW_ENVPROF_W * E->n_envs)); }
  return MW_OK;
}
int mw_get_env_profile(mw_engine* E, unsigned* out) {
  if (!E || !out || !E->d_env_prof) return fail(MW_ERR_STATE, "mw_get_env_profile: profiling is off (mw_set_profiling)");
  CK(cudaSetDevice(E->device));
  CK(cudaMemcpy(out, E->d_env_prof, sizeof(unsigned) * MW_ENVPROF_W * E->n_envs, cudaMemcpyDeviceToHost));
  return MW_OK;
}

int mw_get_env_cost(mw_engine* E, unsigned* out) {
  if (!E || !out || !E->d_env_cost) return fail(MW_ERR_ARG, "mw_get_env_cost");
  CK(cudaSetDevice(E->device));
  CK(cudaMemcpy(out, E->d_env_cost, sizeof(unsigned) * E->n_envs, cudaMemcpyDeviceToHost));
  return MW_OK;
}

int mw_get_profile(mw_engine* E, unsigned long long* out15) {
  if (!E || !out15) return fail(MW_ERR_ARG, "mw_get_profile");
  CK(cudaSetDevice(E->device));
  CK(cudaMemcpy(out15, E->d_prof, sizeof(unsigned long long) * 15, cudaMemcpyDeviceToHost));
  CK(cudaMemset(E->d_prof, 0, sizeof(unsigned long long) * 16));
  return MW_OK;
}

}  // extern "C"
