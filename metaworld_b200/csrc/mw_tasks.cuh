// Per-task device code: observation getters, reward / info, reset_model.
//
// Replaces (reference): SawyerXYZEnv._get_curr_obs_combined_no_goal / _get_obs / step epilogue
// (metaworld/sawyer_xyz_env.py:475-527, 580-642), the shared caging reward (:721-858), reward_utils
// (metaworld/utils/reward_utils.py) and the per-task classes under metaworld/envs/.  Scalar code: it is
// executed by lane 0 of the environment's warp after the physics has left link poses / contacts in the
// warp scratch.  Task ids are the host-side registry order (metaworld_b200/tasks.py).
#pragma once
#include "mw_physics.cuh"

// persistent per-environment record (128 floats = 512 B, one coalesced warp load/store)
struct MwEnvState {
  double qpos[MW_MAXNQ];     // 18 (float64: 36 words; positions carry no per-step float32 rounding)
  float qvel[MW_MAXDOF];     // 17
  float warm[MW_MAXDOF];     // 17
  float mocap_pos[3];
  float prev_obs[18];
  float shift[3];            // run-time translation of the task's movable static body (model.body(..).pos edits)
  float target[3];           // _target_pos
  float obj_init[3];         // obj_init_pos
  float init_tcp[3];
  float scal[16];            // task-specific cached reset constants
  float path_len;            // curr_path_length
  float partially_observable;
  float snapshot;            // snapshot slot this episode started from
  float episode;             // episodes completed (drives the device-side task sampler)
  float ep_return;
  float ended;               // 1: the last step ended the episode and the env has not restarted (NEXT_STEP / DISABLED autoreset)
  float gripper_ctrl;        // last gripper command a[3] (data.ctrl = [a3, -a3]); -1 at episode start (_reset_hand)
  float pad[2];
};
static_assert(sizeof(MwEnvState) == 128 * 4, "MwEnvState must be 128 floats");

struct MwSnapshot { MwEnvState st; float obs[39]; float pad[25]; };
static_assert(sizeof(MwSnapshot) == 192 * 4, "MwSnapshot must be 192 floats");

// per-task constants that are not part of the physics model (host fills from metaworld_b200/tasks.py)
struct MwTaskConst {
  int task_id, nframe_task, main_geom, pad;
  float hand_init[3], mocap_lo[3], mocap_hi[3], goal_lo[3], goal_hi[3], movable_pos0[3];
  float p[16];
};

enum { INFO_SUCCESS = 0, INFO_NEAR_OBJECT, INFO_GRASP_SUCCESS, INFO_GRASP_REWARD, INFO_IN_PLACE, INFO_OBJ_TO_TARGET, INFO_UNSCALED, INFO_N };

// ---- reward utilities (metaworld/utils/reward_utils.py)
// Where the reference raises ValueError (reward_utils.py:124-135 `tolerance`: lower > upper, margin < 0; :237-238
// `hamacher_product`: inputs outside [0, 1]) a kernel cannot: the value is clamped AND the condition is recorded in the
// env's fault word (MW_FAULT_* in include/metaworld_b200.h, read with mw_get_faults), so the host can raise.
#define MW_FAULT_TOL_BOUNDS 1
#define MW_FAULT_TOL_MARGIN 2
#define MW_FAULT_HAMACHER 4
#define MW_FAULT_NONFINITE 8
#define MW_FAULT_STEP_AFTER_END 16   // DISABLED autoreset: an env was stepped after its episode ended (API misuse, not a GPU fault)
#define MW_FAULT_BAD_LOAD 32         // mw_load_states: no saved record of the env's model at the given index (API misuse)
#define MW_FAULT_BAD_GOAL 64         // mw_reset_rows: the env's row has a non-finite goal or observation (API misuse)
DEV real tol_long_tail_f(int* fault, real x, real lo, real hi, real margin) {
  if (lo > hi) *fault |= MW_FAULT_TOL_BOUNDS;
  if (margin < 0) *fault |= MW_FAULT_TOL_MARGIN;
  if (lo <= x && x <= hi) return 1;
  if (margin <= 0) return 0;
  real d = (x < lo ? lo - x : x - hi) / margin;
  real s = d * (real)3.0;             // sqrt(1/0.1 - 1) = 3
  return 1 / (s * s + 1);
}
DEV real tol_gaussian_f(int* fault, real x, real lo, real hi, real margin) {
  if (lo > hi) *fault |= MW_FAULT_TOL_BOUNDS;
  if (margin < 0) *fault |= MW_FAULT_TOL_MARGIN;
  if (lo <= x && x <= hi) return 1;
  if (margin <= 0) return 0;
  real d = (x < lo ? lo - x : x - hi) / margin;
  real s = d * (real)2.145966026289347;   // sqrt(-2 ln 0.1)
  return exp((real)-0.5 * s * s);
}
DEV real hamacher_f(int* fault, real a, real b) {
  if (!(a >= 0 && a <= 1 && b >= 0 && b <= 1)) *fault |= MW_FAULT_HAMACHER;
  a = fmin(fmax(a, (real)0), (real)1); b = fmin(fmax(b, (real)0), (real)1);
  real den = a + b - a * b;
  return den > 0 ? a * b / den : (real)0;
}
// every caller has the task context `c` in scope
#define tol_long_tail(...) tol_long_tail_f(&c.w->fault, __VA_ARGS__)
#define tol_gaussian(...) tol_gaussian_f(&c.w->fault, __VA_ARGS__)
#define hamacher(...) hamacher_f(&c.w->fault, __VA_ARGS__)
DEV real dist3(const real* a, const real* b) { real t[3]; v3sub(t, a, b); return v3norm(t); }

// scipy Rotation.from_matrix(M).as_quat(): xyzw with scipy's branch choice (no sign canonicalisation)
DEV void mat2quat_scipy(const real* M, real* q) {
  real d[4] = {M[0], M[4], M[8], M[0] + M[4] + M[8]};
  int c = 0; for (int i = 1; i < 4; i++) if (d[i] > d[c]) c = i;
  if (c != 3) {
    int i = c, j = (i + 1) % 3, k = (j + 1) % 3;
    q[i] = 1 - d[3] + 2 * M[3 * i + i];
    q[j] = M[3 * j + i] + M[3 * i + j];
    q[k] = M[3 * k + i] + M[3 * i + k];
    q[3] = M[3 * k + j] - M[3 * j + k];
  } else {
    q[0] = M[7] - M[5]; q[1] = M[2] - M[6]; q[2] = M[3] - M[1]; q[3] = 1 + d[3];
  }
  real n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int i = 0; i < 4; i++) q[i] /= n;
}
DEV void frame_mat(const MwModel* m, const WarpScratch* w, int f, real* R) { real q[4]; mw_frame_quat(m, w, f, q); quat2mat(R, q); }

struct TaskCtx {
  const MwModel* m; const MwTaskConst* tc; WarpScratch* w; MwEnvState* s; const real* action; const float* meshvert;
};
DEV void tcp_center(const TaskCtx& c, real* out) {
  real a[3], b[3]; mw_frame_pos(c.m, c.w, F_REE, a); mw_frame_pos(c.m, c.w, F_LEE, b);
  for (int i = 0; i < 3; i++) out[i] = (a[i] + b[i]) * (real)0.5;
}
// touching_object (sawyer_xyz_env.py:401-440): both pads press on the object geom (collider index g)
DEV bool touching_object(const TaskCtx& c, int g, int g_lpad, int g_rpad) {
  real lf = 0, rf = 0;
  for (int i = 0; i < c.w->ncon; i++) {
    const Contact* k = mw_con(c.w, i);
    if (k->row < 0) continue;
    bool hasobj = k->g1 == g || k->g2 == g;
    if (hasobj && (k->g1 == g_lpad || k->g2 == g_lpad)) lf += k->fn;
    if (hasobj && (k->g1 == g_rpad || k->g2 == g_rpad)) rf += k->fn;
  }
  return lf > 0 && rf > 0;
}
// shared caging reward (sawyer_xyz_env.py:721-858)
DEV real gripper_caging_reward(const TaskCtx& c, const real* obj_pos, real obj_radius, real pad_success_thresh,
                               real object_reach_radius, real xz_thresh, real desired_gripper_effort, int density /*0,1=high,2=medium*/) {
  real lp[3], rp[3], tcp[3];
  mw_frame_pos(c.m, c.w, F_LPAD, lp); mw_frame_pos(c.m, c.w, F_RPAD, rp); tcp_center(c, tcp);
  real pad_y[2] = {lp[1], rp[1]}, cag[2];
  for (int i = 0; i < 2; i++) {
    real to_obj = fabs(pad_y[i] - obj_pos[1]), to_init = fabs(pad_y[i] - (real)c.s->obj_init[1]);
    real margin = fabs(to_init - pad_success_thresh);
    cag[i] = tol_long_tail(to_obj, obj_radius, pad_success_thresh, margin);
  }
  real caging_y = hamacher(cag[0], cag[1]);
  real dx = (real)c.s->obj_init[0] - (real)c.s->init_tcp[0], dz = (real)c.s->obj_init[2] - (real)c.s->init_tcp[2];
  real xz_margin = sqrt(dx * dx + dz * dz) - xz_thresh;
  real ex = tcp[0] - obj_pos[0], ez = tcp[2] - obj_pos[2];
  real caging_xz = tol_long_tail(sqrt(ex * ex + ez * ez), 0, xz_thresh, xz_margin);
  real gripper_closed = fmin(fmax((real)0, c.action[3]), desired_gripper_effort) / desired_gripper_effort;
  real caging = hamacher(caging_y, caging_xz);
  real gripping = caging > (real)0.97 ? gripper_closed : (real)0;
  real cg = hamacher(caging, gripping);
  if (density == 1) cg = (cg + caging) / 2;
  if (density == 2) {
    real oi[3] = {c.s->obj_init[0], c.s->obj_init[1], c.s->obj_init[2]}, it[3] = {c.s->init_tcp[0], c.s->init_tcp[1], c.s->init_tcp[2]};
    real reach_margin = fabs(dist3(oi, it) - object_reach_radius);
    real reach = tol_long_tail(dist3(obj_pos, tcp), 0, object_reach_radius, reach_margin);
    cg = (cg + reach) / 2;
  }
  return cg;
}

// task-local caging override shared by push-back / sweep / sweep-into / soccer (e.g. sawyer_push_back_v3.py:160-254);
// `init_left_pad` / `init_right_pad` alias the live pad positions in the reference (sawyer_xyz_env.py:236-237)
DEV real grip_caging(const TaskCtx& c, const real* obj, real obj_radius, real grip_add, real xz_c) {
  real lp[3], rp[3], tcp[3];
  mw_frame_pos(c.m, c.w, F_LPAD, lp); mw_frame_pos(c.m, c.w, F_RPAD, rp); tcp_center(c, tcp);
  real dl = lp[1] - obj[1], dr = obj[1] - rp[1];
  real rm = fabs(fabs(obj[1] - rp[1]) - (real)0.05), lm = fabs(fabs(obj[1] - lp[1]) - (real)0.05);
  real rc = tol_long_tail(dr, obj_radius, (real)0.05, rm), lc = tol_long_tail(dl, obj_radius, (real)0.05, lm);
  real rg = tol_long_tail(dr, obj_radius, obj_radius + grip_add, rm), lg = tol_long_tail(dl, obj_radius, obj_radius + grip_add, lm);
  real ycag = hamacher(rc, lc), ygrip = hamacher(rg, lg);
  real ix = (real)c.s->obj_init[0] - (real)c.s->init_tcp[0], iz = (real)c.s->obj_init[2] - (real)c.s->init_tcp[2];
  real ex = tcp[0] - obj[0], ez = tcp[2] - obj[2];
  real xz = tol_long_tail(sqrt(ex * ex + ez * ez), 0, xz_c, sqrt(ix * ix + iz * iz) - xz_c);
  real caging = hamacher(ycag, xz);
  return (caging + (caging > (real)0.95 ? ygrip : (real)0)) / 2;
}

#include "mw_tasks_gen.cuh"
