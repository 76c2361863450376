/* metaworld_b200.h -- C ABI of the batched Meta-World step engine (libmwb200.so).
 *
 * The reference has no FFI of its own: its hot path is the Python protocol
 * gymnasium.vector.VectorEnv.step/reset over SawyerXYZEnv (metaworld/__init__.py:491-509,
 * metaworld/sawyer_xyz_env.py:580-682) calling MuJoCo's C library.  Each entry point below
 * names the reference call it stands in for.  Plain pointers and sizes only; pointers marked
 * DEV are device pointers owned by the caller (e.g. torch tensors), everything else is host
 * memory.  All functions return 0 on success, a negative mw_status otherwise; the failing call's
 * message is available from mw_last_error().  Calls taking a stream are asynchronous on it.
 */
#ifndef METAWORLD_B200_H
#define METAWORLD_B200_H
#ifdef __cplusplus
extern "C" {
#endif

typedef struct mw_engine mw_engine;

enum mw_status { MW_OK = 0, MW_ERR_CUDA = -1, MW_ERR_ARG = -2, MW_ERR_STATE = -3 };

/* sizes of the blobs the host code must pass (layout generated from metaworld_b200/lower.py) */
int mw_sizeof_model(void);
int mw_sizeof_taskconst(void);
int mw_sizeof_envstate(void);   /* 512 bytes */
int mw_sizeof_snapshot(void);   /* 768 bytes */
const char* mw_last_error(void);
const char* mw_build_info(void); /* "real=float maxcon=80(shared 48) maxefc=344(shared 216) warps_per_block=7 ..." */

/* Construction: what MujocoEnv.__init__ -> MjModel.from_xml_path does per sub-env
 * (metaworld/sawyer_xyz_env.py:53-63), for n_models distinct (model, task) slots.
 *   models      : n_models consecutive MwModel blobs
 *   taskconsts  : n_models consecutive MwTaskConst blobs
 *   meshverts   : per model, hull vertices float[3*nmeshvert[i]] (may be NULL when 0)            */
int mw_create(mw_engine** out, int device, int n_models, const void* models, const void* taskconsts,
              const float* const* meshverts, const int* nmeshvert);
void mw_destroy(mw_engine*);

/* Environment table: env i uses model slot env_model[i]  (make_mt_envs / make_ml_envs building the
 * sub-env list, metaworld/__init__.py:460-604).  Allocates the persistent per-env state.          */
int mw_set_envs(mw_engine*, int n_envs, const int* env_model);

/* Episode-start snapshots.  The reference's reset() = reset_model, mj_resetData, reset_model
 * (2 x 50 x 5 mj_step, metaworld/sawyer_xyz_env.py:664-695) is a pure function of (task, rand_vec,
 * partially_observable) because tasks freeze rand_vec (set_task, :298-318); it is evaluated once per
 * distinct goal by the same device physics and cached.  Appends n snapshots, returns their ids.
 * rand_vec_pass1 (NULL = same as rand_vec): with an UNFROZEN rand_vec (_make_tasks, the goal_hidden / goal_observable
 * envs, metaworld/env_dict.py:144-152) each reset_model pass draws its own vector; the first pass's one survives in
 * whatever the task's reset_model reads before the next kinematics update (e.g. the stale object pose in the reset obs). */
int mw_build_snapshots(mw_engine*, int n, const int* model_idx, const double* rand_vec /*[n,6] float64, as in Task.data*/,
                       const double* rand_vec_pass1 /*[n,6] or NULL*/, const unsigned char* partially_observable,
                       int* snapshot_ids_out);
/* Appends n snapshot records produced elsewhere (mw_get_snapshots of another engine, e.g. the float64 build of this
 * library, or a checkpoint); same record layout, ids returned like mw_build_snapshots.                           */
int mw_append_snapshots(mw_engine*, int n, const void* records, int* snapshot_ids_out);
int mw_num_snapshots(const mw_engine*);
/* copy snapshot records to the host (tests / checkpointing): out = n * mw_sizeof_snapshot() bytes */
int mw_get_snapshots(mw_engine*, int first, int n, void* out);

/* VectorEnv.reset (per-env SawyerXYZEnv.reset with the task chosen by the task-select wrapper,
 * metaworld/wrappers.py:116-119): env_ids[k] (NULL = all envs in order) starts from snapshot_ids[k].
 * obs: DEV float [n, obs_stride] (first 39 columns written).                                        */
int mw_reset(mw_engine*, int n, const int* env_ids /*DEV or NULL*/, const int* snapshot_ids /*DEV*/,
             float* obs /*DEV*/, int obs_stride, void* stream);

/* VectorEnv.step (metaworld/__init__.py:465,491-509 -> SawyerXYZEnv.step, metaworld/sawyer_xyz_env.py:580-642 +
 * TimeLimit + AutoTerminateOnSuccessWrapper, metaworld/wrappers.py:207-230), autoreset as set by mw_set_autoreset_mode
 * (default SAME_STEP).  All arrays DEV, n_envs rows:
 *   actions [n,4] f32; obs [n,obs_stride] f32 (39 written); reward [n] f32; terminated/truncated [n] u8;
 *   info [n,info_stride] f32, columns 0..6 = success, near_object, grasp_success, grasp_reward, in_place_reward,
 *   obj_to_target, unscaled_reward; when info_stride >= 9 also column 7 = reward and column 8 = terminated + 2*truncated
 *   (one packed record per env for a single device->host copy).
 * SAME_STEP: final_obs [n,obs_stride] / final_info [n,8] (7 infos + episode return) are written only for rows whose
 *   episode ended in this call (terminated|truncated), which then restart from next_snapshot[i] (or, when next_snapshot
 *   is NULL, from a snapshot drawn on the device from the env's own goal set, see mw_set_goal_sets).
 * NEXT_STEP: an ending episode reports its terminal observation in obs and its return in final_info column 7 (nothing
 *   else of final_obs / final_info is written); the env is marked as ended.  The next call restarts it as SAME_STEP
 *   would have (same snapshot choice) and reports the reset observation, reward 0, no flags, an all-zero info row
 *   (columns 7 and 8 included); its action is ignored.
 * DISABLED: an ending episode reports its terminal observation and its return (final_info column 7), and the env is
 *   marked as ended.  Stepping an ended env
 *   leaves its state and output rows untouched and sets MW_FAULT_STEP_AFTER_END (restart it with mw_reset_masked).
 * An ended env's warp still runs the physics of the step (its CTA's warps meet at every phase barrier) and discards it:
 *   mw_get_counters counts that pass in env steps [1] and forward passes [4], not in contacts dropped [2] or solver
 *   iterations [3]; it reports no fault other than MW_FAULT_STEP_AFTER_END.                                          */
int mw_step(mw_engine*, const float* actions, float* obs, int obs_stride, float* reward,
            unsigned char* terminated, unsigned char* truncated, float* info, int info_stride, float* final_obs,
            float* final_info, const int* next_snapshot, void* stream);

/* gymnasium.vector.AutoresetMode of mw_step; other values fail with MW_ERR_ARG.  Takes effect at the next launch. */
enum mw_autoreset_mode { MW_AUTORESET_SAME_STEP = 0, MW_AUTORESET_NEXT_STEP = 1, MW_AUTORESET_DISABLED = 2 };
int mw_set_autoreset_mode(mw_engine*, int mode);

/* VectorEnv.reset(options={"reset_mask": mask}): every env with mask[i] != 0 restarts from snapshot_ids[i] (NULL: a
 * snapshot drawn by the device sampler, as in mw_step) and clears its ended mark; its episode counter advances by one, as
 * in an autoreset (mw_reset sets it to 0).  obs row i (not compacted) is written for those envs only.  mask DEV u8 [n_envs],
 * snapshot_ids DEV [n_envs] or NULL, obs DEV float [n_envs, obs_stride].                                             */
int mw_reset_masked(mw_engine*, const unsigned char* mask, const int* snapshot_ids, float* obs, int obs_stride, void* stream);

/* SawyerXYZEnv.evaluate_state(obs, action) (metaworld/sawyer_xyz_env.py:644-656 -> the task's evaluate_state /
 * compute_reward): reward and info of every env's CURRENT physics state for caller-supplied observations and actions.
 * One forward pass (poses, contact forces for touching_object), no state change.  actions DEV [n,4], obs DEV
 * [n,obs_stride], out DEV [n,8] = the 7 info values then the reward.                                              */
int mw_evaluate(mw_engine*, const float* actions, const float* obs, int obs_stride, float* out, void* stream);

/* MujocoEnv.set_state(qpos, qvel) (gymnasium mujoco_env.py; SawyerMocapBase.set_env_state, metaworld/sawyer_xyz_env.py:97-107)
 * for every env with mask[i] != 0: qpos[i, :nq] and qvel[i, :nv] of that env's model become its physics state; columns
 * past nq / nv are ignored.  qvel is ROUNDED TO FLOAT32, the type the state record keeps it in (qpos stays float64).
 * Nothing else of the record changes: mocap, the frame stack (prev_obs), the warm-start qacc, path length, episode
 * counters, return, target, task scalars, snapshot id and the ended mark stay as they are.  The reference's mj_forward is
 * not run: nothing it computes outlives the next step's own forward pass (the warm start is written by the integrator
 * only); mw_observe computes the observation of the new state.  An ended env (NEXT_STEP / DISABLED) may be set; its
 * restart overwrites the state.  mask DEV u8 [n_envs], qpos DEV f64 [n_envs, 18], qvel DEV f64 [n_envs, 17].        */
int mw_set_physics(mw_engine*, const unsigned char* mask, const double* qpos, const double* qvel, void* stream);
/* SawyerMocapBase.get_env_state() (metaworld/sawyer_xyz_env.py:87-95) for every env, on the device and without host
 * synchronisation: qpos DEV f64 [n_envs, 18], qvel DEV f64 [n_envs, 17] (the float32 record widened); columns past the
 * env's nq / nv are zero.                                                                                         */
int mw_get_physics(mw_engine*, double* qpos, double* qvel, void* stream);
/* SawyerXYZEnv._get_obs() (metaworld/sawyer_xyz_env.py:513-527) of the current state for every env with mask[i] != 0:
 * kinematics, then the frame-stacked observation, unclipped as in the reference (step() clips afterwards); like the
 * reference it makes the current frame the env's prev_obs.  obs DEV float [n_envs, obs_stride]: row i (first 39
 * columns) is written for the masked envs only.  A non-finite observation sets MW_FAULT_NONFINITE.                 */
int mw_observe(mw_engine*, const unsigned char* mask, float* obs, int obs_stride, void* stream);

/* Read-only state accessors of SawyerXYZEnv (metaworld/sawyer_xyz_env.py:67-85, 363-473, 529-535) and MujocoEnv's
 * data.body / site / geom(name) poses, for every env with mask[i] != 0, from the env's current state.  Changes nothing:
 * not the record (frame stack, live target), the warm start, the separating-axis hints or any fault bit other than
 * MW_FAULT_NONFINITE (set for a non-finite frame).  Each output may be NULL; rows of unmasked envs are not written.
 *   mask     DEV u8 [n_envs]
 *   frame    DEV f32 [n_envs, 18] or NULL: hand position, gripper distance and the 14 object slots -- bitwise what the next
 *            mw_observe would put into columns 0..17 (unclipped), including the live target refresh of tasks whose
 *            _target_pos aliases a site (basketball); prev_obs is NOT committed.
 *   frames   DEV [n_models, n_frames] 64-byte records {int link, flags; double pos[3], quat[4]} (built by
 *            metaworld_b200/lower.py query_table from (body|site|geom, name) pairs); flags 1 = rides on the env's shift
 *            of the task's movable body, 2 = the name is missing in that model (NaN row), 4 = the position is the env's
 *            _target_pos (basketball's goal site), 8 / 16 = the env's _target_pos / obj_init_pos is added to the position
 *            (sites whose model.site(name).pos reset_model sets); link -2 = relative to the mocap body.
 *   pose     DEV f64 [n_envs, n_frames, 7] or NULL: xpos then the unit quaternion (w, x, y, z) of each named frame.
 *   touch_geom DEV i32 [n_models] and touching DEV u8 [n_envs], both NULL or both given: touching_object(collider
 *            touch_geom[model]) (sawyer_xyz_env.py:401-440; -1 gives 0).  With it the full mj_forward runs (contacts and
 *            constraint forces, the fingers driven by the record's last gripper command, -1 at episode start, as
 *            data.ctrl); without it the kinematics pass only.                                                   */
int mw_query(mw_engine*, const unsigned char* mask, float* frame, const void* frames, int n_frames, double* pose,
             const int* touch_geom, unsigned char* touching, void* stream);

/* metaworld.policies (ENV_POLICY_MAP[name]().get_action(obs), metaworld/policies/__init__.py:76): the scripted expert
 * action of every row, computed as the reference's numpy float64 code does (metaworld_b200/csrc/mw_policies.cuh) and NOT
 * clipped.  Needs no engine: it depends on its inputs only.  task_ids DEV int32 [n] (metaworld_b200/tasks.py TASK_IDS;
 * an id outside [0, 50) gives a NaN row), obs DEV float [n, obs_stride] (columns 0..38 are read: the base observation,
 * one-hot columns after it are ignored), actions DEV float [n, 4].  Fails with MW_ERR_ARG for n < 0, obs_stride < 39 or
 * a NULL pointer when n > 0.                                                                                     */
int mw_expert_actions(const int* task_ids, const float* obs, int obs_stride, int n, float* actions, void* stream);

/* Per-env fault bits accumulated since the last call (host int[n_envs], cleared by the call; synchronises).  The kernel
 * cannot raise where the reference does, so it clamps and flags:
 *   1 MW_FAULT_TOL_BOUNDS  reward_utils.tolerance: lower > upper          (ValueError, reward_utils.py:124-125)
 *   2 MW_FAULT_TOL_MARGIN  reward_utils.tolerance: margin < 0             (ValueError, reward_utils.py:134-135)
 *   4 MW_FAULT_HAMACHER    hamacher_product input outside [0, 1]          (ValueError, reward_utils.py:237-238)
 *   8 MW_FAULT_NONFINITE   non-finite observation or reward (the reference's `_did_see_sim_exception` path)
 *  16 MW_FAULT_STEP_AFTER_END  DISABLED autoreset: stepped after its episode ended, before mw_reset_masked (gymnasium's
 *                              SyncVectorEnv asserts; SawyerXYZEnv.step raises past max_path_length).  API misuse.   */
int mw_get_faults(mw_engine*, int* out);

/* options: max_episode_steps (TimeLimit), terminate_on_success (0/1), device sampler seed */
int mw_set_options(mw_engine*, int max_episode_steps, int terminate_on_success, unsigned long long seed);
/* per-env contiguous range of snapshot ids [first, first+count) used by the device-side task sampler */
int mw_set_goal_sets(mw_engine*, const int* first /*host [n_envs]*/, const int* count /*host [n_envs]*/);

/* raw state access (tests, checkpoint/resume incl. physics state): n_envs * 512 bytes; record = qpos[18] float64, then
 * float32: qvel[17], warm-start qacc[17], mocap_pos[3], prev_obs[18], ..., ended, gripper_ctrl (the last step's a[3],
 * -1 in every snapshot; mw_set_physics leaves it alone; a record saved before the field existed holds 0 there, which
 * only mw_query's touching reads, until the next step), pad[2] (metaworld_b200/engine.py: ENVSTATE_DTYPE)          */
int mw_get_state(mw_engine*, void* out_host);
int mw_set_state(mw_engine*, const void* in_host);
/* debug: run nstep raw physics substeps (mj_step) on every env with fixed ctrl, no reward/obs */
int mw_debug_substeps(mw_engine*, int nstep, const float* ctrl2 /*host [2]*/, void* stream);
/* debug: one forward pass (mj_forward) per env, no state change; dumps per env mw_debug_dump_floats() floats:
 * contacts [MAXCON][12] = dist, pos[3], normal[3], geom1, geom2 (source geom ids), normal force, dim, efc row;
 * then qacc[MAXDOF]; then ncon, nefc, solver iterations.  dump: DEV float [n_envs * mw_debug_dump_floats()] */
int mw_debug_forward(mw_engine*, const float* ctrl2 /*host [2]*/, float* dump, void* stream);
int mw_debug_dump_floats(void);
/* counters accumulated since the last call: [0] kernel launches, [1] env steps, [2] contacts dropped,
 * [3] solver iterations (sum over forward passes), [4] forward passes */
int mw_get_counters(mw_engine*, unsigned long long* out5);

/* Re-sorts the CTA launch order by the measured mean step cost of each model slot (costliest first), so that the tail of
 * every launch is filled by cheap environments.  Results are unaffected (environments are independent).  Host-synchronising;
 * call it after a few warm-up steps and then rarely.                                                                */
int mw_rebalance(mw_engine*);

/* Profiling switch (default off: the timed kernel then carries no profiling atomics).  When on, mw_step additionally sums
 * the per-phase counters below, the per-model cost used by mw_rebalance, and records per env [20] u32: the 13 counters of
 * mw_get_profile for that env's last step, [13] solver iterations, [14] / [15] largest contact / constraint-row
 * count over the 6 passes, [16] launch slot (CTA), [17] convex candidate pairs queued, [18] / [19] counters [13] / [14] of
 * mw_get_profile for the convex pairs this env's warp evaluated.  Stands in for nothing in the reference (it has no profiler hook on this path).  */
int mw_set_profiling(mw_engine*, int on);
int mw_get_env_profile(mw_engine*, unsigned* out /*host [n_envs*20]*/);

/* per-phase SM cycle counters summed over all env steps since the last call (one warp = one env, so these are
 * warp-cycles): [0] kinematics + mass matrix, [1] collision (incl. [2]), [2] GJK/EPA pairs, [3] constraint rows,
 * [4] bias forces + unconstrained solve, [5] constraint solver, [6] integration + glue, [7] obs / reward / autoreset,
 * [8] whole step incl. [12]; events: [9] GJK/EPA pair calls, [10] EPA expansions, [11] GJK iterations; [12] cycles spent
 * waiting for the CTA's other warps at phase boundaries (not part of [0]..[7]); [13] GJK/EPA pairs tested against their
 * separating-axis hint, [14] of those, pairs the hint proved apart (no GJK/EPA run; [2] and [9] include them) */
int mw_get_profile(mw_engine*, unsigned long long* out15);
/* warp cycles each environment spent in its most recent step (host array of n_envs) */
int mw_get_env_cost(mw_engine*, unsigned* out);

#ifdef __cplusplus
}
#endif
#endif
