// One-environment-per-warp forward dynamics + semi-implicit Euler step.
//
// Hot path replaced: the reference's `do_simulation` -> `mujoco.mj_step(nstep=5)` and `mj_forward`
// (metaworld/sawyer_xyz_env.py:595,620) -- MuJoCo's CPU pipeline [3P] -- for the Meta-World MJCF
// feature set.  A warp owns one environment for the whole env step (5 substeps + 1 forward), so the
// state makes a single HBM round trip; all intermediates live in the warp's shared-memory scratch.
//
// Lane mapping: lane d <-> degree of freedom d (nv <= 17) for Jacobian columns, inertia columns and
// dense vectors; lane r <-> constraint row / contact for per-row work; lane p <-> candidate pair in the
// broadphase / analytic narrowphase.  Reductions are warp shuffles in a fixed order (deterministic).
#pragma once
#include "mw_model.h"
#include "mw_collide.cuh"

#define NVP 17               // row stride of the dense nv x nv / nefc x nv matrices (odd: conflict-free columns)
// Capacities.  The warp's shared-memory scratch holds MW_SMCON contacts and MW_SMEFC constraint rows: enough for all but
// ~1e-4 of env steps (p99.99 of the per-step contact maximum is 37).  An env that exceeds them in some pass - a jam: e.g. a
// plug wedged in its socket with 6 box-box pairs x 8 points - is NOT truncated: contacts MW_SMCON.. and rows MW_SMEFC.. go to
// a per-warp global-memory block (WarpSpill) and that pass runs the <SP = true> instantiation of the constraint code, which
// addresses rows / contacts through a storage selector.  Same arithmetic, same order: results do not depend on where a row
// lives (checked by building with tiny shared capacities and comparing digests, scripts/gpu_ab.py).  Only beyond MW_MAXCON /
// MW_MAXEFC is a contact dropped, and counted.
#ifndef MW_SMCON
#define MW_SMCON 48
#endif
#ifndef MW_MAXCON
#define MW_MAXCON 80
#endif
#define MW_MAXSCALAR 24      // weld (6) + joint-limit rows
#define MW_SMEFC (MW_MAXSCALAR + 4 * MW_SMCON)     // every shared-memory contact can be condim 4
#define MW_MAXEFC (MW_MAXSCALAR + 4 * MW_MAXCON)

enum { JT_FREE = 0, JT_BALL, JT_SLIDE, JT_HINGE };

struct ConvRes { RawCon r; int hit, pad; };   // result slot of one convex candidate pair (written by whichever warp of the CTA processed it)

struct Contact {
  real pos[3], frame[9], dist, mu, fr1, fr3;
  real H[10];              // packed symmetric dim x dim cone Hessian (row-major upper)
  real fn;                 // normal force of the last solve
  short row, prm;          // first efc row (-1: not instantiated), index into MwModel.param (margin, solref, solimp ...)
  unsigned char dim, g1, g2, hzone;
};

// region U is time-shared: (a) geom world poses + EPA workspace during collision, (b) efc_J afterwards
#define MW_UWORDS_J (MW_SMEFC * NVP)
#define MW_UWORDS_C (MW_MAXGEOM * 12 * 2 + (int)(sizeof(EpaSm) / 4) + 2 + MW_MAXCAND * (int)(sizeof(ConvRes) / 4))   // geom world poses (creal) + EPA scratch + convex-pair results during collision
#define MW_UWORDS (MW_UWORDS_J > MW_UWORDS_C ? MW_UWORDS_J : MW_UWORDS_C)

// CTA-wide sharing of the general convex pairs (GJK/EPA): every warp publishes its env's candidate pairs, then all warps
// of the CTA pull (env, pair) items from one queue, so one env with many penetrating mesh pairs does not hold up its CTA
// (and the kernel: the slowest env's collision phase was the critical path of the whole step).
#define MW_MAXCAND 48
struct CtaShare { int q_head, nwarp, peer_stride, pad; unsigned char* peer0; int q_cnt[16]; };

struct WarpSpill;

struct WarpScratch {
  real lpos[MW_MAXLINK][3], lquat[MW_MAXLINK][4], lmat[MW_MAXLINK][9];
  real lcom[MW_MAXLINK][3], lIw[MW_MAXLINK][9];   // world COM and world inertia about it (mw_link_inertia; read by mw_mass_matrix, mw_rne_bias)
  real daxis[MW_MAXDOF][3], danchor[MW_MAXDOF][3];
  real qpos[MW_MAXNQ], qvel[MW_MAXDOF], warm[MW_MAXDOF];
  // positions are carried in float64 (state record, kinematic chain, collision inputs): float32 storage of qpos was the
  // largest per-step noise source (6e-8 relative, every step); qpos[] above is the float copy the dynamics reads
  double qposd[MW_MAXNQ], lposd[MW_MAXLINK][3], lquatd[MW_MAXLINK][4];
  real ctrl[2], mocap_pos[3], mocap_quat[4], shift[3];
  real qfrc_smooth[MW_MAXDOF], qacc_smooth[MW_MAXDOF], qfrc_con[MW_MAXDOF], qacc[MW_MAXDOF];
  real vMa[MW_MAXDOF], vSearch[MW_MAXDOF], vMs[MW_MAXDOF], vTmp[MW_MAXDOF];
  real M[MW_MAXDOF * NVP], H[MW_MAXDOF * NVP];
  alignas(16) real U[MW_UWORDS];
  EpaWs* epa;               // this warp's GJK/EPA polytope workspace (global memory, see mw_engine.cu)
  WarpSpill* sp;            // overflow storage for contacts >= MW_SMCON / rows >= MW_SMEFC (global memory)
  float4* sep;              // this env's MW_NCONV separating-axis hints, by pair_cslot (global memory; null: no hints)
  real eD[MW_SMEFC], eAref[MW_SMEFC], eJar[MW_SMEFC], eJv[MW_SMEFC], eF[MW_SMEFC], eHd[MW_MAXSCALAR];
  Contact con[MW_SMCON];
  unsigned short cand[MW_MAXCAND];   // this env's general convex candidate pairs of the current pass (pair indices)
  unsigned char achunk[MW_MAXCON];   // 32-pair chunk each analytic contact came from (contact order, see mw_collide)
  CtaShare* cta; int warp_in_cta, ncand;
  int nblk1;                // mw_tree_split of the model: dofs [0, nblk1) and [nblk1, nv) never share a kinematic tree
  int ncon, nefc, nscalar, nweld, solver_iter, ncon_dropped;
  int fault;                // MW_FAULT_* bits raised by the task code during this step (lane 0)
  int prof_on;              // phase timers enabled (mw_set_profiling)
  long long prof[16];       // cycle / event counters of this step (mw_get_profile order; [12] = cycles spent waiting in PHASE_SYNC,
                            // [13] / [14] = convex pairs tested against / rejected by their separating-axis hint; lane 0 only)
};

struct WarpSpill {
  real J[(MW_MAXEFC - MW_SMEFC) * NVP];
  real eD[MW_MAXEFC - MW_SMEFC], eAref[MW_MAXEFC - MW_SMEFC], eJar[MW_MAXEFC - MW_SMEFC], eJv[MW_MAXEFC - MW_SMEFC], eF[MW_MAXEFC - MW_SMEFC];
  Contact con[MW_MAXCON - MW_SMCON];
};
// storage selectors (used by the SP = true instantiations and by the few cold call sites that may see any contact index)
DEV real* mw_jrow(const WarpScratch* w, int r) { return r < MW_SMEFC ? (real*)w->U + r * NVP : w->sp->J + (r - MW_SMEFC) * NVP; }
DEV real* mw_ev(const real* sm, real* gl, int r) { return r < MW_SMEFC ? (real*)sm + r : gl + (r - MW_SMEFC); }
DEV Contact* mw_con(const WarpScratch* w, int c) { return c < MW_SMCON ? (Contact*)&w->con[c] : &w->sp->con[c - MW_SMCON]; }
// inside `template <bool SP>` functions: direct shared-memory addressing unless this pass overflowed
#define JROW(r) (SP ? mw_jrow(w, (r)) : (real*)w->U + (r) * NVP)
#define EV(name, r) (*(SP ? mw_ev(w->name, w->sp->name, (r)) : (real*)&w->name[r]))
#define CON(c) (SP ? mw_con(w, (c)) : (Contact*)&w->con[c])

#define SYNCW() __syncwarp()
// cycle counter that the compiler may not move across barriers / memory operations (plain clock64() was hoisted above
// __syncthreads(), which booked every barrier wait on the phase that follows it)
DEV long long mw_clock() { long long t; asm volatile("mov.u64 %0, %%clock64;" : "=l"(t) :: "memory"); return t; }
// Reading the clock is not free (ncu: 5.7 % of all stall samples sat on the ~80 reads per env step), so the phase timers
// only run while profiling is switched on (mw_set_profiling); MW_CLK(w) is 0 otherwise.
#define MW_CLK(w) ((w)->prof_on ? mw_clock() : 0ll)
#define QSET(w, i, v) { (w)->qposd[i] = (double)(v); (w)->qpos[i] = (real)(w)->qposd[i]; }   /* write a generalized position */

// ------------------------------------------------------------------ kinematics  [MuJoCo mj_kinematics]
// Sequential over the (short) link chain; every lane computes the same values, lane 0 stores.
__device__ __noinline__ void mw_kinematics(const MwModel* __restrict__ m, WarpScratch* w, int lane) {
  const int nl = m->nlink;
  double quat[4], R[9];          // orientation of the link in work; at the top of an iteration: of the previous link
  for (int l = 0; l < nl; l++) {
    int p = m->link_parent[l];
    double pos[3];
    if (p < 0) {
      if (m->link_shift[l]) { for (int i = 0; i < 3; i++) pos[i] = (double)m->link_pos[l][i] + (double)w->shift[i]; }
      else { for (int i = 0; i < 3; i++) pos[i] = m->link_pos[l][i]; }
      for (int i = 0; i < 4; i++) quat[i] = m->link_quat[l][i];
    } else {
      double lp[3] = {m->link_pos[l][0], m->link_pos[l][1], m->link_pos[l][2]};
      double lq[4] = {m->link_quat[l][0], m->link_quat[l][1], m->link_quat[l][2], m->link_quat[l][3]};
      // the arm is a chain: the parent is usually the previous link, whose matrix and quaternion are still in registers
      double Rp[9], pq[4], t[3];
      if (p == l - 1) { for (int i = 0; i < 9; i++) Rp[i] = R[i]; for (int i = 0; i < 4; i++) pq[i] = quat[i]; }
      else { for (int i = 0; i < 4; i++) pq[i] = w->lquatd[p][i]; quat2mat(Rp, pq); }
      mat_mulvec(t, Rp, lp); v3add(pos, w->lposd[p], t);
      quat_mul(quat, pq, lq);
    }
    const int jt = m->link_jtype[l], qa = m->link_qadr[l], da = m->link_dadr[l];
    bool fresh = false;          // `quat` has just been normalised and R is its matrix
    if (jt == JT_FREE) {
      double q[4] = {w->qposd[qa + 3], w->qposd[qa + 4], w->qposd[qa + 5], w->qposd[qa + 6]};
      quat_normalize(q);
      for (int i = 0; i < 3; i++) pos[i] = w->qposd[qa + i];
      for (int i = 0; i < 4; i++) quat[i] = q[i];
      quat2mat(R, quat); fresh = true;
      if (lane == 0) {
        for (int i = 0; i < 4; i++) QSET(w, qa + 3 + i, q[i]);
        for (int i = 0; i < 3; i++) {
          for (int k = 0; k < 3; k++) { w->daxis[da + i][k] = (i == k); w->danchor[da + i][k] = (real)pos[k]; }
          w->daxis[da + 3 + i][0] = (real)R[i]; w->daxis[da + 3 + i][1] = (real)R[3 + i]; w->daxis[da + 3 + i][2] = (real)R[6 + i];
          for (int k = 0; k < 3; k++) w->danchor[da + 3 + i][k] = (real)pos[k];
        }
      }
    } else {
      double jax[3] = {m->link_jaxis[l][0], m->link_jaxis[l][1], m->link_jaxis[l][2]};
      double jp[3] = {m->link_jpos[l][0], m->link_jpos[l][1], m->link_jpos[l][2]};
      double axis[3], anchor[3], t[3];
      // joint axis and anchor in the frame the body has before its own joint moves it (a product of unit quaternions:
      // like mj_kinematics, no normalisation before the end of the body)
      quat2mat(R, quat);
      mat_mulvec(axis, R, jax);
      mat_mulvec(t, R, jp); v3add(anchor, pos, t);
      double q = w->qposd[qa] - m->qpos0d[qa];
      if (jt == JT_SLIDE) v3addscl(pos, pos, axis, q);
      else {
        double qr[4], qn[4];
        quat_axisangle(qr, jax, q);
        quat_mul(qn, quat, qr);
        for (int i = 0; i < 4; i++) quat[i] = qn[i];
        quat_normalize(quat);
        quat2mat(R, quat); fresh = true;
        mat_mulvec(t, R, jp); v3sub(pos, anchor, t);
      }
      if (lane == 0) for (int k = 0; k < 3; k++) { w->daxis[da][k] = (real)axis[k]; w->danchor[da][k] = (real)anchor[k]; }
    }
    if (!fresh) { quat_normalize(quat); quat2mat(R, quat); }
    if (lane == 0) {
      for (int i = 0; i < 3; i++) { w->lposd[l][i] = pos[i]; w->lpos[l][i] = (real)pos[i]; }
      for (int i = 0; i < 4; i++) { w->lquatd[l][i] = quat[i]; w->lquat[l][i] = (real)quat[i]; }
      for (int i = 0; i < 9; i++) w->lmat[l][i] = (real)R[i];
    }
    SYNCW();
  }
}

// world pose of a frame / geom attached to link l (or to the world, optionally riding on the shift)
DEV void mw_attach(const WarpScratch* w, int link, int shift, const float* lp, real* pos) {
  real p[3] = {lp[0], lp[1], lp[2]};
  if (link < 0) { for (int i = 0; i < 3; i++) pos[i] = p[i] + (shift ? w->shift[i] : (real)0); }
  else { real t[3]; mat_mulvec(t, w->lmat[link], p); v3add(pos, w->lpos[link], t); }
}
DEV void mw_frame_pos(const MwModel* m, const WarpScratch* w, int f, real* pos) {
  mw_attach(w, m->frame_link[f], m->frame_shift[f], m->frame_pos[f], pos);
}
DEV void mw_frame_quat(const MwModel* m, const WarpScratch* w, int f, real* q) {
  real fq[4] = {m->frame_quat[f][0], m->frame_quat[f][1], m->frame_quat[f][2], m->frame_quat[f][3]};
  int l = m->frame_link[f];
  if (l < 0) { for (int i = 0; i < 4; i++) q[i] = fq[i]; }
  else quat_mul(q, w->lquat[l], fq);
  quat_normalize(q);
}

// per-lane dof description held in registers
struct LaneDof { real ax[3], an[3]; int rot; int valid; };
DEV void mw_lane_dof(const MwModel* m, const WarpScratch* w, int lane, LaneDof* L) {
  L->valid = lane < m->nv;
  int d = L->valid ? lane : 0;
  for (int k = 0; k < 3; k++) { L->ax[k] = L->valid ? w->daxis[d][k] : (real)0; L->an[k] = w->danchor[d][k]; }
  int l = m->dof_link[d];
  int jt = m->link_jtype[l];
  L->rot = (jt == JT_HINGE) || (jt == JT_FREE && (d - m->link_dadr[l]) >= 3);
}
// column `lane` of the Jacobian of a world point on a body whose ancestor-dof mask is `mask`
DEV void mw_jac_col(const LaneDof& L, unsigned mask, int lane, const real* point, real* jp, real* jr) {
  if (L.valid && ((mask >> lane) & 1u)) {
    if (L.rot) { real r[3]; v3sub(r, point, L.an); v3cross(jp, L.ax, r); v3copy(jr, L.ax); }
    else { v3copy(jp, L.ax); v3zero(jr); }
  } else { v3zero(jp); v3zero(jr); }
}

// World COM and world inertia about the COM (R I R^T) of every link, one link per lane (every lane used to repeat this for
// every link, once for the mass matrix and once more for the bias forces).
DEV void mw_link_inertia_one(const MwModel* __restrict__ m, const WarpScratch* w, int l, real* c, real* Iw) {
  const real* R = w->lmat[l];
  real cl[3] = {m->link_com[l][0], m->link_com[l][1], m->link_com[l][2]}, t[3];
  mat_mulvec(t, R, cl); v3add(c, w->lpos[l], t);
  real I6[6] = {m->link_inertia[l][0], m->link_inertia[l][1], m->link_inertia[l][2], m->link_inertia[l][3], m->link_inertia[l][4], m->link_inertia[l][5]};
  real Il[9] = {I6[0], I6[3], I6[4], I6[3], I6[1], I6[5], I6[4], I6[5], I6[2]}, T[9];
  mat_mul(T, R, Il);
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Iw[3 * i + j] = T[3 * i] * R[3 * j] + T[3 * i + 1] * R[3 * j + 1] + T[3 * i + 2] * R[3 * j + 2];
}
DEV void mw_link_inertia(const MwModel* __restrict__ m, WarpScratch* w, int lane) {
  const int l = lane;
  if (l < m->nlink && m->link_mass[l] > 0) {
    real c[3], Iw[9];
    mw_link_inertia_one(m, w, l, c, Iw);
    for (int i = 0; i < 3; i++) w->lcom[l][i] = c[i];
    for (int i = 0; i < 9; i++) w->lIw[l][i] = Iw[i];
  }
  SYNCW();
}

// ------------------------------------------------------------------ inertia  [MuJoCo mj_crb]
// M = sum_links S^T I_link S with spatial vectors about the world origin; lane d owns column d.
__device__ __noinline__ void mw_mass_matrix(const MwModel* __restrict__ m, WarpScratch* w, const LaneDof& L, int lane) {
  const int nv = m->nv;
  for (int i = lane; i < nv * NVP; i += 32) w->M[i] = 0;
  SYNCW();
  real Sa[3], Sl[3];   // spatial motion vector of this lane's dof
  if (L.rot) { v3copy(Sa, L.ax); v3cross(Sl, L.an, L.ax); } else { v3zero(Sa); v3copy(Sl, L.ax); }
  if (!L.valid) { v3zero(Sa); v3zero(Sl); }
  mw_link_inertia(m, w, lane);
  for (int l = 0; l < m->nlink; l++) {
    real mass = m->link_mass[l];
    if (mass <= 0) continue;
    unsigned mask = m->link_dofmask[l];
    real c[3], t[3], Iw[9];
    for (int i = 0; i < 3; i++) c[i] = w->lcom[l][i];
    for (int i = 0; i < 9; i++) Iw[i] = w->lIw[l][i];
    // momentum of this lane's dof: p = m (v + w x c), Lang = Iw w + c x p
    real pl[3], La[3];
    v3cross(t, Sa, c); for (int i = 0; i < 3; i++) pl[i] = mass * (Sl[i] + t[i]);
    mat_mulvec(La, Iw, Sa); v3cross(t, c, pl); v3add(La, La, t);
    bool mine = L.valid && ((mask >> lane) & 1u);
    unsigned rem = mask;
    while (rem) {
      int e = __ffs(rem) - 1; rem &= rem - 1;
      real ea[3] = {bcast(Sa[0], e), bcast(Sa[1], e), bcast(Sa[2], e)};
      real el[3] = {bcast(Sl[0], e), bcast(Sl[1], e), bcast(Sl[2], e)};
      if (mine) w->M[e * NVP + lane] += v3dot(ea, La) + v3dot(el, pl);
    }
  }
  if (L.valid) w->M[lane * NVP + lane] += m->dof_armature[lane];
  SYNCW();
}

// number of leading dofs that form the kinematic tree of dof 0 (the arm in 46 of the 50 models, the mug's free joint in
// the coffee models): M is block diagonal over kinematic trees, and so is H = M + J^T D J unless a contact row touches both
DEV int mw_tree_split(const MwModel* __restrict__ m) {
  unsigned blk = 0;
  for (int l = 0; l < m->nlink; l++) if (m->link_dofmask[l] & 1u) blk |= m->link_dofmask[l];
  const int nb = __ffs(~blk) - 1;                      // length of the run of low set bits
  return (blk >> nb) != 0 || nb <= 0 ? m->nv : nb;     // the tree's dofs are not a prefix: no split
}

// in-place Cholesky of the lower triangle of A (stride NVP); lane i owns row i.
// Right-looking with the lane's row held in registers (fully unrolled to MW_MAXDOF, guarded by the trip count): column j is
// scaled, broadcast by shuffles and subtracted from the trailing columns; every element receives its updates in increasing
// column order, so the factor is bit-identical to the left-looking dot-product form.
// TWO CHAINS: the factorisation is a dependent chain of nv columns (shuffle -> sqrt -> divide -> shuffle -> fma per column)
// and that latency, not the instruction count, is its cost.  When the block A[nb.., ..nb) is exactly zero (always for M and
// M + hB, and for H whenever no active contact couples the two trees) the two diagonal blocks are independent problems:
// lanes < nb factor block 1 while lanes >= nb factor block 2 in the same instruction stream (each lane keeps its row
// shifted to its block's first column), max(nb, nv - nb) columns instead of nv.  The skipped work is exclusively
// `x -= l * 0` on the zero block, so the result equals the single-chain factor bit for bit.  One copy of the code
// (__noinline__; it is 17 KB and used to be inlined at three call sites).  Returns the split that was used (nv: one chain)
// for mw_chol_solve.
// x / d for d > 0 without the division's slow path when x is exactly zero (right-hand sides are full of exact zeros: a
// resting object's dofs); the result is the same zero
DEV real mw_div_nz(real x, real d) { const real q = (x != (real)0 ? x : (real)1) / d; return x != (real)0 ? q : x; }
// (a value the compiler can prove warp-uniform: without it every guarded shuffle is wrapped in divergence handling)
DEV int mw_uniform(int v, int lane) { return __popc(__ballot_sync(FULLMASK, lane < v)); }
// columns 0 .. NM-1 of the lane's block.  Columns / rows a block does not have need no guard: no lane has `row >= j` for
// them, so every update is predicated off (the shuffles are harmless).
template <int NM> DEV void mw_chol_cols(real* A, int lane, int off, int row, int ncol) {
  real a[NM];
#pragma unroll
  for (int k = 0; k < NM; k++) a[k] = k <= row ? A[lane * NVP + off + k] : (real)0;
#pragma unroll
  for (int j = 0; j < NM; j++) {
    if (NM <= 10 || j < ncol) {                                  // (uniform; the short variant runs straight through)
      real piv = __shfl_sync(FULLMASK, a[j], off + j);
      piv = sqrt(fmax(piv, (real)1e-30));
      // (a zero numerator sends the IEEE division to its slow path -- a 30-instruction subroutine on the factorisation's
      // critical chain -- and most lanes hold one: rows above the pivot, structural zeros of the block.  0 / piv = 0 with
      // the sign of the zero, so those lanes divide 1 instead and keep their zero)
      const real aj = a[j];
      const bool dv = row > j && aj != (real)0;
      const real qt = (dv ? aj : (real)1) / piv;
      const real lij = row == j ? piv : (dv ? qt : (row > j ? aj : (real)0));  // L[off + row][off + j]
      a[j] = lij;
#pragma unroll
      for (int k = j + 1; k < NM; k++) {
        const real lkj = __shfl_sync(FULLMASK, lij, off + k);  // L[off + k][off + j]
        if (k <= row) a[k] -= lij * lkj;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < NM; k++) if (k <= row) A[lane * NVP + off + k] = a[k];
}
__device__ __noinline__ int mw_chol(real* A, int nv, int nb, int lane) {
  if (nb < nv) {
    bool cpl = false;
    if (lane >= nb && lane < nv) for (int k = 0; k < nb; k++) cpl |= A[lane * NVP + k] != (real)0;
    if (__any_sync(FULLMASK, cpl)) nb = nv;
  }
  const int off = lane < nb ? 0 : nb;                  // first dof of this lane's block
  const int row = lane < nv ? lane - off : -1;         // row inside the block (lanes beyond nv hold nothing)
  const int nmax = mw_uniform(nb > nv - nb ? nb : nv - nb, lane);
  if (nmax <= 10) mw_chol_cols<10>(A, lane, off, row, nmax);          // every model's blocks have <= 10 dofs
  else mw_chol_cols<MW_MAXDOF>(A, lane, off, row, nmax);              // one chain (coupled H, or a model without a split)
  SYNCW();
  return nb;
}
// solve L L^T x = b ; lane i holds b_i / returns x_i.  `nb` is the split mw_chol returned: the substitutions of the two
// blocks run side by side (2 max(nb, nv - nb) dependent steps instead of 2 nv; same arithmetic per element).
// (A fully unrolled variant with the lane's row and column of L in registers, the counterpart of mw_chol_cols, was measured
// slower per env step -- identical results -- and is not used.)
DEV real mw_chol_solve(const real* Lm, real b, int nv, int nb, int lane) {
  const int off = lane < nb ? 0 : nb, end = lane < nb ? nb : nv;
  const int nmax = mw_uniform(nb > nv - nb ? nb : nv - nb, lane);
  real y = b;
  for (int j = 0; j < nmax; j++) {
    const int c = off + j; const bool in = c < end; const int cc = in ? c : 0;
    real xj = mw_div_nz(__shfl_sync(FULLMASK, y, cc), Lm[cc * NVP + cc]);
    if (in) {
      if (lane == c) y = xj;
      else if (lane > c && lane < end) y -= Lm[lane * NVP + c] * xj;
    }
  }
  for (int j = nmax - 1; j >= 0; j--) {
    const int c = off + j; const bool in = c < end; const int cc = in ? c : 0;
    real xj = mw_div_nz(__shfl_sync(FULLMASK, y, cc), Lm[cc * NVP + cc]);
    if (in) {
      if (lane == c) y = xj;
      else if (lane < c && lane >= off) y -= Lm[c * NVP + lane] * xj;
    }
  }
  return lane < nv ? y : (real)0;
}

// ------------------------------------------------------------------ bias forces  [MuJoCo mj_comVel + mj_rne]
DEV void cross_motion(real* r, const real* v, const real* s) {
  real a[3], b[3], c[3];
  v3cross(a, v, s); v3cross(b, v, s + 3); v3cross(c, v + 3, s);
  r[0] = a[0]; r[1] = a[1]; r[2] = a[2]; r[3] = b[0] + c[0]; r[4] = b[1] + c[1]; r[5] = b[2] + c[2];
}
// returns qfrc_bias for this lane's dof.  Uses w->H as scratch (cvel/cacc/cfrc per link).
__device__ __noinline__ real mw_rne_bias(const MwModel* __restrict__ m, WarpScratch* w, const LaneDof& L, int lane) {
  real* cvel = w->H; real* cacc = w->H + 6 * MW_MAXLINK; real* cfrc = w->H + 12 * MW_MAXLINK;
  const int nl = m->nlink;
  for (int l = 0; l < nl; l++) {
    int p = m->link_parent[l];
    real v[6], a[6];
    if (p < 0) { for (int c = 0; c < 6; c++) { v[c] = 0; a[c] = 0; } a[3] = -m->gravity[0]; a[4] = -m->gravity[1]; a[5] = -m->gravity[2]; }
    else { for (int c = 0; c < 6; c++) { v[c] = cvel[6 * p + c]; a[c] = cacc[6 * p + c]; } }
    int jt = m->link_jtype[l], da = m->link_dadr[l];
    if (jt == JT_FREE) {
      real vb[6];
      for (int i = 0; i < 3; i++) {   // world-fixed translation axes
        real S[6] = {0, 0, 0, w->daxis[da + i][0], w->daxis[da + i][1], w->daxis[da + i][2]}, Sd[6];
        cross_motion(Sd, v, S);
        real qd = w->qvel[da + i];
        for (int c = 0; c < 6; c++) { a[c] += Sd[c] * qd; }
        for (int c = 0; c < 6; c++) v[c] += S[c] * qd;
      }
      for (int c = 0; c < 6; c++) vb[c] = v[c];
      for (int i = 3; i < 6; i++) {   // body-fixed rotation axes: all three see the same velocity
        real S[6], Sd[6];
        for (int k = 0; k < 3; k++) S[k] = w->daxis[da + i][k];
        v3cross(S + 3, w->danchor[da + i], w->daxis[da + i]);
        cross_motion(Sd, vb, S);
        real qd = w->qvel[da + i];
        for (int c = 0; c < 6; c++) { a[c] += Sd[c] * qd; v[c] += S[c] * qd; }
      }
    } else {
      real S[6], Sd[6];
      if (jt == JT_HINGE) { for (int k = 0; k < 3; k++) S[k] = w->daxis[da][k]; v3cross(S + 3, w->danchor[da], w->daxis[da]); }
      else { S[0] = S[1] = S[2] = 0; for (int k = 0; k < 3; k++) S[3 + k] = w->daxis[da][k]; }
      cross_motion(Sd, v, S);
      real qd = w->qvel[da];
      for (int c = 0; c < 6; c++) { v[c] += S[c] * qd; a[c] += Sd[c] * qd; }
    }
    // body force f = I a + v x* (I v)
    real mass = m->link_mass[l];
    real f[6] = {0, 0, 0, 0, 0, 0};
    if (mass > 0) {
      real c[3], t[3], u[3], Iw[9];      // from mw_link_inertia (mw_mass_matrix ran on the same poses)
      for (int i = 0; i < 3; i++) c[i] = w->lcom[l][i];
      for (int i = 0; i < 9; i++) Iw[i] = w->lIw[l][i];
      real pl[3], Lm[3], pa[3], La[3];
      v3cross(t, v, c); for (int i = 0; i < 3; i++) pl[i] = mass * (v[3 + i] + t[i]);
      mat_mulvec(Lm, Iw, v); v3cross(t, c, pl); v3add(Lm, Lm, t);
      v3cross(t, a, c); for (int i = 0; i < 3; i++) pa[i] = mass * (a[3 + i] + t[i]);
      mat_mulvec(La, Iw, a); v3cross(t, c, pa); v3add(La, La, t);
      v3cross(t, v, Lm); v3cross(u, v + 3, pl);
      for (int i = 0; i < 3; i++) f[i] = La[i] + t[i] + u[i];
      v3cross(t, v, pl);
      for (int i = 0; i < 3; i++) f[3 + i] = pa[i] + t[i];
    }
    if (lane == 0) for (int c = 0; c < 6; c++) { cvel[6 * l + c] = v[c]; cacc[6 * l + c] = a[c]; cfrc[6 * l + c] = f[c]; }
    SYNCW();
  }
  // leaves-to-root accumulation of the link forces: the six components are independent, one lane each
  if (lane < 6) for (int l = nl - 1; l >= 0; l--) { int p = m->link_parent[l]; if (p >= 0) cfrc[6 * p + lane] += cfrc[6 * l + lane]; }
  SYNCW();
  real bias = 0;
  if (L.valid) {
    const real* f = cfrc + 6 * m->dof_link[lane];
    real Sa[3], Sl[3];
    if (L.rot) { v3copy(Sa, L.ax); v3cross(Sl, L.an, L.ax); } else { v3zero(Sa); v3copy(Sl, L.ax); }
    bias = v3dot(Sa, f) + v3dot(Sl, f + 3);
  }
  SYNCW();
  return bias;
}

// ------------------------------------------------------------------ collision  [MuJoCo mj_collision]
DEV void mw_load_shape(const MwModel* m, const creal* gpose, const float* meshvert, int g, DShape* s) {
  s->type = m->geom_type[g];
  s->pos = gpose + 12 * g; s->mat = gpose + 12 * g + 3;
  for (int i = 0; i < 3; i++) s->size[i] = m->geom_size[g][i];
  s->vert = (const float4*)meshvert + m->geom_meshadr[g]; s->nvert = m->geom_meshnum[g];
}
DEV void make_frame(creal* fr) {
  v3normalize(fr);
  creal* y = fr + 3; creal* z = fr + 6;
  v3zero(y);
  if (fr[1] < (creal)0.5 && fr[1] > (creal)-0.5) y[1] = 1; else y[2] = 1;
  creal dp = v3dot(fr, y);
  v3addscl(y, y, fr, -dp);
  v3normalize(y);
  v3cross(z, fr, y);
}
DEV void mw_store_contact(const MwModel* m, WarpScratch* w, int slot, const RawCon& rc, int pair) {
  Contact* c = mw_con(w, slot);
  int prm = m->pair_param[pair];
  const float* P = m->param[prm];
  c->dist = (real)rc.dist;
  creal fr[9] = {rc.normal[0], rc.normal[1], rc.normal[2], 0, 0, 0, 0, 0, 0};
  make_frame(fr);
  for (int k = 0; k < 3; k++) c->pos[k] = (real)rc.pos[k];
  for (int k = 0; k < 9; k++) c->frame[k] = (real)fr[k];
  c->g1 = m->pair_g1[pair]; c->g2 = m->pair_g2[pair];
  c->prm = (short)prm; c->dim = (unsigned char)P[2]; c->fr1 = P[3]; c->fr3 = P[4]; c->mu = P[3];
  c->row = -1; c->fn = 0; c->hzone = 0;
  w->achunk[slot] = (unsigned char)(pair >> 5);
}

__device__ __noinline__ void mw_collide(const MwModel* __restrict__ m, const float* __restrict__ meshvert, WarpScratch* w, int lane) {
  creal* gpose = (creal*)w->U;                          // [ngeom][12] world poses, float64 from here on
  EpaWs* epa = w->epa;
  EpaSm* esm = (EpaSm*)(gpose + MW_MAXGEOM * 12);
  const int ng = m->ngeom, np = m->npair;
  for (int g = lane; g < ng; g += 32) {
    const int l = m->geom_link[g];
    creal gp[3] = {m->geom_pos[g][0], m->geom_pos[g][1], m->geom_pos[g][2]}, pos[3];
    creal Rl[9]; for (int i = 0; i < 9; i++) Rl[i] = m->geom_mat[g][i];
    creal Rw[9];
    if (l < 0) {
      for (int i = 0; i < 3; i++) pos[i] = gp[i] + (m->geom_shift[g] ? (creal)w->shift[i] : (creal)0);
      for (int i = 0; i < 9; i++) Rw[i] = Rl[i];
    } else {
      creal Lm[9], Lp[3], t[3];
      quat2mat(Lm, w->lquatd[l]);
      for (int i = 0; i < 3; i++) Lp[i] = w->lposd[l][i];
      mat_mulvec(t, Lm, gp); v3add(pos, Lp, t);
      mat_mul(Rw, Lm, Rl);
    }
    for (int i = 0; i < 3; i++) gpose[12 * g + i] = pos[i];
    for (int i = 0; i < 9; i++) gpose[12 * g + 3 + i] = Rw[i];
  }
  if (lane == 0) { w->ncon = 0; w->ncon_dropped = 0; }
  SYNCW();
  int ncon = 0, ncand = 0, nover = 0;
  for (int base = 0; base < np; base += 32) {
    int p = base + lane;
    // ---- broadphase cull (conservative: never removes a pair that is within margin)
    bool keep = false; int g1 = 0, g2 = 0; creal margin = 0;
    if (p < np) {
      g1 = m->pair_g1[p]; g2 = m->pair_g2[p];
      margin = m->param[m->pair_param[p]][0];
      int t1 = m->geom_type[g1], t2 = m->geom_type[g2];
      const creal* p1 = gpose + 12 * g1; const creal* p2 = gpose + 12 * g2;
      creal r1 = m->geom_rbound[g1], r2 = m->geom_rbound[g2];
      if (t1 == G_PLANE) {
        creal n[3], t[3]; mat_col(n, p1 + 3, 2); v3sub(t, p2, p1);
        keep = v3dot(t, n) <= r2 + margin;
      } else {
        creal t[3]; v3sub(t, p2, p1);
        creal bound = r1 + r2 + margin;
        keep = v3dot(t, t) <= bound * bound;
        // bounding sphere of one geom against the oriented bounding box of the other (exact for boxes, hull extents for meshes)
        if (keep) {
          const float* bb = m->geom_aabb[g2];
          creal cl[3], dd = 0; mat_tmulvec(cl, p2 + 3, t);     // centre of g1 in the frame of g2 is -R2^T t
          for (int i = 0; i < 3; i++) { creal e = fabs(-cl[i] - (creal)bb[i]) - (creal)bb[3 + i]; if (e > 0) dd += e * e; }
          creal b = r1 + margin; keep = dd <= b * b;
        }
        if (keep) {
          const float* bb = m->geom_aabb[g1];
          creal cl[3], dd = 0; mat_tmulvec(cl, p1 + 3, t);      // centre of g2 in the frame of g1 is +R1^T t
          for (int i = 0; i < 3; i++) { creal e = fabs(cl[i] - (creal)bb[i]) - (creal)bb[3 + i]; if (e > 0) dd += e * e; }
          creal b = r2 + margin; keep = dd <= b * b;
        }
      }
    }
    // ---- analytic pairs: one pair per lane
    bool analytic = keep && pair_is_analytic(m->geom_type[g1], m->geom_type[g2]);
    RawCon rc[8]; int cnt = 0;
    if (analytic) {
      DShape a, b; mw_load_shape(m, gpose, meshvert, g1, &a); mw_load_shape(m, gpose, meshvert, g2, &b);
      cnt = narrow_analytic(a, b, margin, rc);
    } else if (keep && m->geom_type[g1] == G_CYLINDER && (m->geom_type[g2] == G_BOX || m->geom_type[g2] == G_CYLINDER)) {
      // axis-aligned cylinder-box / parallel cylinders: exact, one pair per lane; anything else falls through to GJK/EPA
      DShape a, b; mw_load_shape(m, gpose, meshvert, g1, &a); mw_load_shape(m, gpose, meshvert, g2, &b);
      const int r = b.type == G_BOX ? cyl_box_aligned(a, b, margin, rc) : cyl_cyl_parallel(a, b, margin, rc);
      if (r >= 0) { cnt = r; analytic = true; }
    }
    // deterministic compaction: exclusive prefix of counts over lanes
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(FULLMASK, incl, o); if (lane >= o) incl += t; }
    int start = ncon + incl - cnt;
    for (int k = 0; k < cnt; k++) if (start + k < MW_MAXCON) mw_store_contact(m, w, start + k, rc[k], p);
    ncon += __shfl_sync(FULLMASK, incl, 31);
    // ---- general convex pairs (cylinder / mesh): deferred to the CTA-wide queue below
    unsigned cm = __ballot_sync(FULLMASK, keep && !analytic);
    while (cm) {
      int src = __ffs(cm) - 1; cm &= cm - 1;
      if (ncand < MW_MAXCAND) { if (lane == 0) w->cand[ncand] = (unsigned short)(base + src); ncand++; }
      else nover++;
    }
  }
  ConvRes* cres = (ConvRes*)((unsigned char*)esm + sizeof(EpaSm));
  CtaShare* cs = w->cta;
  if (lane == 0) { w->ncand = ncand; cs->q_cnt[w->warp_in_cta] = ncand; }
  if (threadIdx.x == 0) cs->q_head = 0;
  __syncthreads();                       // candidates of all envs of the CTA are published
  {
    const int nw = cs->nwarp;
    int total = 0; for (int o = 0; o < nw; o++) total += cs->q_cnt[o];
    for (;;) {
      int item = 0;
      if (lane == 0) item = atomicAdd(&cs->q_head, 1);
      item = __shfl_sync(FULLMASK, item, 0);
      if (item >= total) break;
      int o = 0, k = item;
      while (k >= cs->q_cnt[o]) { k -= cs->q_cnt[o]; o++; }
      WarpScratch* ow = (WarpScratch*)(cs->peer0 + (size_t)o * cs->peer_stride);     // the env this pair belongs to (same model: same CTA)
      const creal* ogpose = (const creal*)ow->U;
      ConvRes* ores = (ConvRes*)((unsigned char*)ogpose + MW_MAXGEOM * 12 * sizeof(creal) + sizeof(EpaSm));
      const int pp = ow->cand[k];
      int h1 = m->pair_g1[pp], h2 = m->pair_g2[pp];
      DShape a, b; mw_load_shape(m, ogpose, meshvert, h1, &a); mw_load_shape(m, ogpose, meshvert, h2, &b);
      creal mg = m->param[m->pair_param[pp]][0];
      RawCon r1; int c1;
      if (a.type == G_PLANE) {   // plane - mesh: support vertex against the plane
        creal n[3], nd[3], sp[3], t[3]; mat_col(n, a.mat, 2); v3scl(nd, n, -1);
        support_shape(b, nd, sp, lane);
        v3sub(t, sp, a.pos);
        r1.dist = v3dot(t, n); v3copy(r1.normal, n); v3addscl(r1.pos, sp, n, -(creal)0.5 * r1.dist);
        c1 = r1.dist <= mg;
      } else {
        const long long tc = MW_CLK(w);
        float4* hint = nullptr;
#ifndef MW_NO_SEPCACHE
        if (ow->sep && m->pair_cslot[pp] < MW_NCONV) hint = ow->sep + m->pair_cslot[pp];
#endif
        // a pair the owner's hint still proves apart skips GJK/EPA; its result is the one GJK would give (sep_hint_test)
        const int ht = hint ? sep_hint_test(a, b, mg, hint, lane) : -1;
        c1 = ht == 1 ? 0 : convex_pair(a, b, mg, &r1, esm, epa, lane, w->prof, hint);
        if (lane == 0) {
          w->prof[2] += MW_CLK(w) - tc; w->prof[9] += 1;
          if (w->prof_on) { w->prof[13] += ht >= 0; w->prof[14] += ht == 1; }
        }
      }
      if (lane == 0) { ores[k].hit = c1; if (c1) ores[k].r = r1; }
    }
  }
  __syncthreads();                       // all results are in their owners' slots
  // Merge the convex hits into the contact list.  Order (a pure function of the state, identical to the order the pairs
  // were visited in when every warp ran its own convex pairs inline): 32-pair chunk by chunk, within a chunk the analytic
  // contacts first, then the convex ones in pair order.  Walk from the back so nothing is overwritten before it is moved.
  {
    int nhit = 0;
    for (int k = 0; k < ncand; k++) nhit += cres[k].hit != 0;
    const int nA = ncon < MW_MAXCON ? ncon : MW_MAXCON;      // analytic contacts actually stored
    int j = nA + nhit - 1, ai = nA - 1, hk = ncand - 1;
    SYNCW();
    while (nhit > 0 && j >= 0) {
      while (hk >= 0 && !cres[hk].hit) hk--;
      const bool take_hit = hk >= 0 && (ai < 0 || (int)w->achunk[ai] <= (int)(w->cand[hk] >> 5));
      if (take_hit) {
        if (j < MW_MAXCON && lane == 0) mw_store_contact(m, w, j, cres[hk].r, w->cand[hk]);
        hk--; nhit--;
      } else {
        if (j < MW_MAXCON && j != ai) {
          const unsigned* src = (const unsigned*)mw_con(w, ai); unsigned* dst = (unsigned*)mw_con(w, j);
          for (int q = lane; q < (int)(sizeof(Contact) / 4); q += 32) dst[q] = src[q];
          if (lane == 0) w->achunk[j] = w->achunk[ai];
        }
        ai--;
      }
      j--;
      SYNCW();
    }
    for (int k = 0; k < ncand; k++) ncon += cres[k].hit != 0;
  }
  SYNCW();
  if (lane == 0) { w->ncon = ncon < MW_MAXCON ? ncon : MW_MAXCON; w->ncon_dropped = (ncon > MW_MAXCON ? ncon - MW_MAXCON : 0) + nover; }
  SYNCW();
}

// ------------------------------------------------------------------ constraint rows  [MuJoCo mj_makeConstraint]
struct RowParam { real K, B, imp; };
DEV RowParam mw_impedance(real pos_minus_margin, const real* solref, const real* solimp, real timestep) {
  real lo = fmin(fmax(solimp[0], (real)0.0001), (real)0.9999), hi = fmin(fmax(solimp[1], (real)0.0001), (real)0.9999);
  real width = fmax(solimp[2], (real)0), mid = fmin(fmax(solimp[3], (real)0.0001), (real)0.9999), power = fmax(solimp[4], (real)1);
  real imp;
  if (lo == hi || width <= MW_EPS) imp = (real)0.5 * (lo + hi);
  else {
    real x = fabs(pos_minus_margin) / width;
    if (x >= 1) imp = hi;
    else if (x <= 0) imp = lo;
    else {
      real y;
      if (power == 1) y = x;
      else if (x <= mid) y = pow(x, power) / pow(mid, power - 1);
      else y = 1 - pow(1 - x, power) / pow(1 - mid, power - 1);
      imp = lo + y * (hi - lo);
    }
  }
  RowParam r; r.imp = imp;
  if (solref[0] > 0) {
    real tc = fmax(solref[0], 2 * timestep), dr = solref[1];
    r.K = 1 / fmax(MW_EPS, hi * hi * tc * tc * dr * dr);
    r.B = 2 / fmax(MW_EPS, hi * tc);
  } else { r.K = -solref[0] / fmax(MW_EPS, hi * hi); r.B = -solref[1] / fmax(MW_EPS, hi); }
  return r;
}

template <bool SP> __device__ __noinline__ void mw_make_constraints(const MwModel* __restrict__ m, WarpScratch* w, const LaneDof& L, int lane) {
  const int nv = m->nv;
  const real h = m->timestep;
  // ---- weld rows 0..5 (mocap -> hand)
  int wl = m->weld_link;
  real ph[3], qh[4];
  { real wp[3] = {m->weld_pos[0], m->weld_pos[1], m->weld_pos[2]}, t[3]; mat_mulvec(t, w->lmat[wl], wp); v3add(ph, w->lpos[wl], t);
    real wq[4] = {m->weld_quat[0], m->weld_quat[1], m->weld_quat[2], m->weld_quat[3]}; quat_mul(qh, w->lquat[wl], wq); }
  real qm[4] = {w->mocap_quat[0], w->mocap_quat[1], w->mocap_quat[2], w->mocap_quat[3]};
  quat_normalize(qm);
  real q[4] = {-qm[0], -qm[1], -qm[2], -qm[3]};            // q_mocap * relpose(-1,0,0,0)
  real q1n[4] = {qh[0], -qh[1], -qh[2], -qh[3]}, q2[4];
  quat_mul(q2, q1n, q);
  const real ts = m->weld_torquescale;
  real cpos[6] = {w->mocap_pos[0] - ph[0], w->mocap_pos[1] - ph[1], w->mocap_pos[2] - ph[2], ts * q2[1], ts * q2[2], ts * q2[3]};
  {
    real jp[3], jr[3];
    mw_jac_col(L, m->link_dofmask[wl], lane, ph, jp, jr);
    real axq[4] = {0, -jr[0], -jr[1], -jr[2]}, a4[4], b4[4];
    quat_mul(a4, q1n, axq); quat_mul(b4, a4, q);
    if (lane < nv) for (int k = 0; k < 3; k++) { JROW(k)[lane] = -jp[k]; JROW(3 + k)[lane] = (real)0.5 * ts * b4[1 + k]; }
  }
  int nrow = 6;
  // ---- joint limits
  bool lim_lo = false, lim_hi = false; real ldist = 0;
  if (L.valid && m->dof_limited[lane]) {
    real qv = w->qpos[m->dof_qadr[lane]];
    real dlo = qv - m->dof_lo[lane], dhi = m->dof_hi[lane] - qv;
    if (dlo < 0) { lim_lo = true; ldist = dlo; } else if (dhi < 0) { lim_hi = true; ldist = dhi; }
  }
  unsigned lm = __ballot_sync(FULLMASK, lim_lo || lim_hi);
  int nlim = __popc(lm);
  if (nrow + nlim > MW_MAXSCALAR) { nlim = MW_MAXSCALAR - nrow; }
  int myrank = __popc(lm & ((1u << lane) - 1));
  for (int r = 0; r < nlim; r++) if (lane < nv) JROW(nrow + r)[lane] = 0;
  SYNCW();
  if ((lim_lo || lim_hi) && myrank < nlim) JROW(nrow + myrank)[lane] = lim_lo ? (real)1 : (real)-1;
  // per-row scalars for limit rows are filled below by the owning dof lane
  const int nscalar = nrow + nlim;
  // ---- contact rows
  int nefc = nscalar;
  const int ncon = w->ncon;
  for (int c = 0; c < ncon; c++) {
    Contact* con = CON(c);
    if (con->dist >= (real)m->param[con->prm][1]) { if (lane == 0) con->row = -1; continue; }
    if (nefc + con->dim > MW_MAXEFC) { if (lane == 0) { con->row = -1; w->ncon_dropped++; } continue; }   // counted, reported by mw_get_counters
    int l1 = m->geom_link[con->g1], l2 = m->geom_link[con->g2];
    unsigned m1 = l1 < 0 ? 0u : m->link_dofmask[l1], m2 = l2 < 0 ? 0u : m->link_dofmask[l2];
    real p[3] = {con->pos[0], con->pos[1], con->pos[2]};
    real jp1[3], jr1[3], jp2[3], jr2[3];
    mw_jac_col(L, m1, lane, p, jp1, jr1);
    mw_jac_col(L, m2, lane, p, jp2, jr2);
    real dp[3], dr[3]; v3sub(dp, jp2, jp1); v3sub(dr, jr2, jr1);
    if (lane < nv) {
      for (int k = 0; k < 3; k++) JROW(nefc + k)[lane] = v3dot(con->frame + 3 * k, dp);
      if (con->dim > 3) JROW(nefc + 3)[lane] = v3dot(con->frame, dr);
    }
    if (lane == 0) con->row = nefc;
    nefc += con->dim;
  }
  SYNCW();
  // ---- per-row scalars: weld (lanes 0..5), limits (owning dof lane), contacts (lane c)
  if (lane < 6) {
    real vel = 0; for (int k = 0; k < nv; k++) vel += JROW(lane)[k] * w->qvel[k];
    real sr[2] = {m->weld_solref[0], m->weld_solref[1]}, si[5] = {m->weld_solimp[0], m->weld_solimp[1], m->weld_solimp[2], m->weld_solimp[3], m->weld_solimp[4]};
    RowParam rp = mw_impedance(cpos[lane], sr, si, h);
    real diag = lane < 3 ? m->weld_invw[0] : m->weld_invw[1];
    real Rr = fmax(MW_EPS, (1 - rp.imp) * diag / rp.imp);
    EV(eD, lane) = 1 / Rr;
    EV(eAref, lane) = -rp.B * vel - rp.K * rp.imp * cpos[lane];
  }
  if ((lim_lo || lim_hi) && myrank < nlim) {
    int r = nrow + myrank;
    real vel = (lim_lo ? (real)1 : (real)-1) * w->qvel[lane];
    real sr[2] = {(real)0.02, (real)1}, si[5] = {(real)0.9, (real)0.95, (real)0.001, (real)0.5, (real)2};
    RowParam rp = mw_impedance(ldist, sr, si, h);
    real Rr = fmax(MW_EPS, (1 - rp.imp) * m->dof_invweight[lane] / rp.imp);
    EV(eD, r) = 1 / Rr;
    EV(eAref, r) = -rp.B * vel - rp.K * rp.imp * ldist;
  }
  for (int ci = lane; ci < ncon; ci += 32) {
    Contact* con = CON(ci);
    if (con->row < 0) continue;
    int r0 = con->row, dim = con->dim;
    real tran = m->geom_invw[con->g1][0] + m->geom_invw[con->g2][0];
    real rot = m->geom_invw[con->g1][1] + m->geom_invw[con->g2][1];
    const float* Pm = m->param[con->prm];
    const real incl = Pm[1], solref[2] = {Pm[5], Pm[6]}, solimp[5] = {Pm[7], Pm[8], Pm[9], Pm[10], Pm[11]};
    RowParam rp = mw_impedance(con->dist - incl, solref, solimp, h);
    RowParam rf = mw_impedance((real)0, solref, solimp, h);
    real R0 = fmax(MW_EPS, (1 - rp.imp) * tran / rp.imp);
    (void)rot;
    real R1 = R0 / m->impratio;
    con->mu = con->fr1 * sqrt(R1 / R0);
    const real Rk[4] = {R0, R1, R1, R1 * con->fr1 * con->fr1 / (con->fr3 * con->fr3)};
#pragma unroll
    for (int k = 0; k < 4; k++) if (k < dim) {
      real vel = 0; for (int d = 0; d < nv; d++) vel += JROW(r0 + k)[d] * w->qvel[d];
      EV(eD, r0 + k) = 1 / Rk[k];
      EV(eAref, r0 + k) = k == 0 ? (-rp.B * vel - rp.K * rp.imp * (con->dist - incl)) : (-rf.B * vel);
    }
  }
  if (lane == 0) { w->nefc = nefc; w->nscalar = nscalar; w->nweld = 6; }
  SYNCW();
}

// ------------------------------------------------------------------ constraint cost / force / Hessian blocks
// scalar rows on lanes [0,nscalar), contacts on lanes [0,ncon) (two passes); x = jar (+ alpha*jv).
template <bool SP> DEV real mw_scalar_row(const WarpScratch* w, int r, real x, real* f, real* hd) {
  real D = EV(eD, r);
  bool active = (r < w->nweld) || x < 0;
  *f = active ? -D * x : (real)0; *hd = active ? D : (real)0;
  return active ? (real)0.5 * D * x * x : (real)0;
}
// elliptic cone block; x[0..dim) ; optionally forces and packed Hessian.  All loops run to the fixed bound 4 with a
// `k < dim` guard and are fully unrolled: the small arrays then live in registers instead of the thread's local-memory
// stack (dynamically indexed arrays were the bulk of the kernel's 5.9 K LDL/STL instructions and of its DRAM traffic).
template <bool SP> DEV real mw_cone(const WarpScratch* w, const Contact* con, const real* x, real* f, real* Hc, int* zone) {
  const int r0 = con->row, dim = con->dim;
  const real mu = con->mu;
  const real fr[4] = {0, con->fr1, con->fr1, con->fr3};
  real u[4] = {0, 0, 0, 0};
  real N = x[0] * mu, T2 = 0;
#pragma unroll
  for (int k = 1; k < 4; k++) if (k < dim) { u[k] = x[k] * fr[k]; T2 += u[k] * u[k]; }
  real T = sqrt(T2), cost = 0;
  if (Hc) {
#pragma unroll
    for (int i = 0; i < 10; i++) Hc[i] = 0;
  }
  if (N >= mu * T || (T <= 0 && N >= 0)) {
    *zone = 0;
    if (f) {
#pragma unroll
      for (int k = 0; k < 4; k++) f[k] = 0;
    }
  } else if (mu * N + T <= 0 || (T <= 0 && N < 0)) {
    *zone = 1;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int dg = k == 0 ? 0 : (k == 1 ? 4 : (k == 2 ? 7 : 9));
      if (k < dim) {
        real Dk = EV(eD, r0 + k);
        cost += (real)0.5 * Dk * x[k] * x[k];
        if (f) f[k] = -Dk * x[k];
        if (Hc) Hc[dg] = Dk;
      } else if (f) f[k] = 0;
    }
  } else {
    *zone = 2;
    real Dm = EV(eD, r0) / fmax(MW_EPS, mu * mu * (1 + mu * mu));
    real NmT = N - mu * T;
    cost = (real)0.5 * Dm * NmT * NmT;
    real g[4] = {mu, 0, 0, 0};
#pragma unroll
    for (int k = 1; k < 4; k++) if (k < dim) g[k] = -mu * fr[k] * u[k] / T;
    if (f) {
#pragma unroll
      for (int k = 0; k < 4; k++) f[k] = k < dim ? -Dm * NmT * g[k] : (real)0;
    }
    if (Hc) {
      real s = -Dm * NmT * mu, iT = 1 / T, iT3 = iT * iT * iT;
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = a; b < 4; b++) {
          const int idx = a == 0 ? b : (a == 1 ? 3 + b : (a == 2 ? 5 + b : 9));   // packed upper-triangular index of (a, b)
          if (a < dim && b < dim) {
            real hv = Dm * g[a] * g[b];
            if (a >= 1) { real t2 = -(fr[a] * u[a]) * (fr[b] * u[b]) * iT3; if (a == b) t2 += fr[a] * fr[a] * iT; hv += s * t2; }
            Hc[idx] = hv;
          }
        }
    }
  }
  return cost;
}
// full evaluation at jar: returns total constraint cost; stores forces (eF), scalar Hessian diag (eHd) and cone Hessians
template <bool SP> DEV real mw_constraint_eval(WarpScratch* w, int lane, bool want_hess) {
  real cost = 0;
  if (lane < w->nscalar) { real f, hd; cost += mw_scalar_row<SP>(w, lane, EV(eJar, lane), &f, &hd); EV(eF, lane) = f; w->eHd[lane] = hd; }
  for (int ci = lane; ci < w->ncon; ci += 32) {
    Contact* con = CON(ci);
    if (con->row < 0) continue;
    real x[4] = {0, 0, 0, 0}, f[4]; int zone;
    const int cdim = con->dim, crow = con->row;
#pragma unroll
    for (int k = 0; k < 4; k++) if (k < cdim) x[k] = EV(eJar, crow + k);
    cost += mw_cone<SP>(w, con, x, f, want_hess ? con->H : nullptr, &zone);
#pragma unroll
    for (int k = 0; k < 4; k++) if (k < cdim) EV(eF, crow + k) = f[k];
    con->hzone = zone; con->fn = f[0];
  }
  return warp_sum(cost);
}
template <bool SP> DEV void mw_linesearch_eval(const WarpScratch* w, int lane, real alpha, real* c, real* g, real* hh) {
  real cc = 0, gg = 0, h2 = 0;
  if (lane < w->nscalar) {
    real jv = EV(eJv, lane), x = EV(eJar, lane) + alpha * jv, D = EV(eD, lane);
    if (lane < w->nweld || x < 0) { cc += (real)0.5 * D * x * x; gg += D * x * jv; h2 += D * jv * jv; }
  }
  for (int ci = lane; ci < w->ncon; ci += 32) {
    const Contact* con = CON(ci);
    if (con->row < 0) continue;
    const int r0 = con->row, dim = con->dim; const real mu = con->mu;
    const real fr[4] = {0, con->fr1, con->fr1, con->fr3};
    real jvk[4] = {0, 0, 0, 0}, xk4[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 4; k++) if (k < dim) { jvk[k] = EV(eJv, r0 + k); xk4[k] = EV(eJar, r0 + k) + alpha * jvk[k]; }
    real N = xk4[0] * mu, Np = jvk[0] * mu, T2 = 0, xv = 0, vv = 0;
#pragma unroll
    for (int k = 1; k < 4; k++) if (k < dim) {
      real fk = fr[k], jv = jvk[k], xk = xk4[k];
      T2 += fk * fk * xk * xk; xv += fk * fk * xk * jv; vv += fk * fk * jv * jv;
    }
    real T = sqrt(T2);
    if (N >= mu * T || (T <= 0 && N >= 0)) {
    } else if (mu * N + T <= 0 || (T <= 0 && N < 0)) {
#pragma unroll
      for (int k = 0; k < 4; k++) if (k < dim) {
        real Dk = EV(eD, r0 + k), jv = jvk[k], xk = xk4[k];
        cc += (real)0.5 * Dk * xk * xk; gg += Dk * xk * jv; h2 += Dk * jv * jv;
      }
    } else {
      real Dm = EV(eD, r0) / fmax(MW_EPS, mu * mu * (1 + mu * mu));
      real NmT = N - mu * T, Tp = xv / T, Tpp = vv / T - xv * xv / (T * T * T);
      real r = Np - mu * Tp;
      cc += (real)0.5 * Dm * NmT * NmT; gg += Dm * NmT * r; h2 += Dm * (r * r - NmT * mu * Tpp);
    }
  }
  *c = warp_sum(cc); *g = warp_sum(gg); *hh = warp_sum(h2);
}

// y_lane = sum_k A[lane][k] x_k  (x published through vTmp)
// A is the mass matrix: block diagonal over the kinematic trees by construction (mw_mass_matrix only ever touches pairs
// of dofs of one tree), so a row's sum runs over its own block; the skipped terms are exact zeros times x_k.
DEV real mw_matvec(const real* A, WarpScratch* w, real x, int nv, int lane) {
  if (lane < nv) w->vTmp[lane] = x;
  SYNCW();
  real s = 0;
  const int nb = w->nblk1, k0 = lane < nb ? 0 : nb, k1 = lane < nb ? nb : nv;
  if (lane < nv) for (int k = k0; k < k1; k++) s += A[lane * NVP + k] * w->vTmp[k];
  SYNCW();
  return s;
}
// rows of J times a dof vector held in vTmp -> out[r]
template <bool SP> DEV void mw_J_times(const WarpScratch* w, real* out_sm, real* out_gl, int nefc, int nv, int lane) {
  for (int r = lane; r < nefc; r += 32) {
    real s = 0;
    for (int k = 0; k < nv; k++) s += JROW(r)[k] * w->vTmp[k];
    *(SP ? mw_ev(out_sm, out_gl, r) : out_sm + r) = s;
  }
}

// ------------------------------------------------------------------ solver  [MuJoCo mj_solNewton, primal]
// minimise 1/2 (a-a0)^T M (a-a0) + s(J a - aref).  Newton with exact Hessian + exact 1-D line search.
template <bool SP> __device__ __noinline__ void mw_solve(const MwModel* __restrict__ m, WarpScratch* w, int lane, int max_iter) {
  const int nv = m->nv, nefc = w->nefc;
  const real scale = m->solver_scale;
  const real tol = sizeof(real) == 4 ? (real)1e-7 : (real)1e-10;
  const real qfs = lane < nv ? w->qfrc_smooth[lane] : (real)0;
  const real a0 = lane < nv ? w->qacc_smooth[lane] : (real)0;
  // ---- warm start selection  [mj_warmstart]
  real qacc = 0, Ma = 0, cost = 0;
  bool warm_won = true;
  for (int pass = 0; pass < 2; pass++) {
    real a = lane < nv ? (pass == 0 ? w->warm[lane] : a0) : (real)0;
    real Maa = mw_matvec(w->M, w, a, nv, lane);
    if (lane < nv) w->vTmp[lane] = a;
    SYNCW();
    mw_J_times<SP>(w, w->eJar, w->sp->eJar, nefc, nv, lane);
    SYNCW();
    for (int r = lane; r < nefc; r += 32) EV(eJar, r) -= EV(eAref, r);
    SYNCW();
    real gauss = warp_sum((real)0.5 * (a - a0) * (Maa - qfs));
    real c = gauss + mw_constraint_eval<SP>(w, lane, false);
    SYNCW();
    if (pass == 0 || c < cost) { cost = c; qacc = a; Ma = Maa; warm_won = pass == 0; }
  }
  if (warm_won) {     // eJar currently holds J a0 - aref (the second candidate): rebuild it for the warm start that won
    if (lane < nv) w->vTmp[lane] = qacc;
    SYNCW();
    mw_J_times<SP>(w, w->eJar, w->sp->eJar, nefc, nv, lane);
    SYNCW();
    for (int r = lane; r < nefc; r += 32) EV(eJar, r) -= EV(eAref, r);
    SYNCW();
  }
  int iter = 0;
  for (; iter < max_iter; iter++) {
    // forces + Hessian blocks at the current point
    mw_constraint_eval<SP>(w, lane, true);
    SYNCW();
    // gradient
    real grad = 0;
    if (lane < nv) { grad = Ma - qfs; for (int r = 0; r < nefc; r++) grad -= JROW(r)[lane] * EV(eF, r); }
    real gn = sqrt(warp_sum(grad * grad));
    if (scale * gn < tol) break;
    // H = M + J^T Hblocks J : lane b owns column b, lower triangle a >= b.  The column is accumulated in registers (fully
    // unrolled over the rows with guards, the Jacobian entries arrive as shared-memory broadcasts) and stored once; every
    // element receives its terms in the same order as a read-modify-write loop over shared memory would give it.
    {
      real h[MW_MAXDOF];
      const bool own = lane < nv;
#pragma unroll
      for (int a = 0; a < MW_MAXDOF; a++) h[a] = (own && a >= lane && a < nv) ? w->M[a * NVP + lane] : (real)0;
      for (int r = 0; r < w->nscalar; r++) {
        const real hd = w->eHd[r];
        if (hd == 0) continue;
        const real* Jr = JROW(r);
        const real wb = own ? hd * Jr[lane] : (real)0;
        const bool on = wb != 0;
#pragma unroll
        for (int a = 0; a < MW_MAXDOF; a++) if (a < nv) { const real ja = Jr[a]; if (on && a >= lane) h[a] += ja * wb; }
      }
      for (int c = 0; c < w->ncon; c++) {
        const Contact* con = CON(c);
        if (con->row < 0 || con->hzone == 0) continue;
        const int r0 = con->row, dim = con->dim;
        // dofs that can move either body: every other column of these rows is exactly zero, so skipping them adds nothing
        const int cl1 = m->geom_link[con->g1], cl2 = m->geom_link[con->g2];
        const unsigned cmask = (cl1 < 0 ? 0u : m->link_dofmask[cl1]) | (cl2 < 0 ? 0u : m->link_dofmask[cl2]);
        const bool on = own && ((cmask >> lane) & 1u);
        real Jb[4] = {0, 0, 0, 0}, t[4];
        const real* J0 = JROW(r0); const real* J1 = JROW(r0 + 1); const real* J2 = JROW(r0 + 2); const real* J3 = JROW(r0 + 3);
        const int ln = own ? lane : 0;
        Jb[0] = J0[ln]; if (dim > 1) Jb[1] = J1[ln]; if (dim > 2) Jb[2] = J2[ln]; if (dim > 3) Jb[3] = J3[ln];
        // t = Hc * Jb (packed symmetric upper, row-major 4x4; entries beyond dim are zero)
        const real* Hc = con->H;
        const real h0 = Hc[0], h1 = Hc[1], h2 = Hc[2], h3 = Hc[3], h4 = Hc[4], h5 = Hc[5], h6 = Hc[6], h7 = Hc[7], h8 = Hc[8], h9 = Hc[9];
        t[0] = h0 * Jb[0] + h1 * Jb[1] + h2 * Jb[2] + h3 * Jb[3];
        t[1] = h1 * Jb[0] + h4 * Jb[1] + h5 * Jb[2] + h6 * Jb[3];
        t[2] = h2 * Jb[0] + h5 * Jb[1] + h7 * Jb[2] + h8 * Jb[3];
        t[3] = h3 * Jb[0] + h6 * Jb[1] + h8 * Jb[2] + h9 * Jb[3];
#pragma unroll
        for (int a = 0; a < MW_MAXDOF; a++) {
          if ((cmask >> a) & 1u) {                       // (uniform: the contact is the same for every lane)
            real s = J0[a] * t[0];
            if (dim > 1) s += J1[a] * t[1];
            if (dim > 2) s += J2[a] * t[2];
            if (dim > 3) s += J3[a] * t[3];
            if (on && a >= lane) h[a] += s;
          }
        }
      }
#pragma unroll
      for (int a = 0; a < MW_MAXDOF; a++) if (own && a >= lane && a < nv) w->H[a * NVP + lane] = h[a];
    }
    SYNCW();
    const int nbe = mw_chol(w->H, nv, w->nblk1, lane);
    real search = -mw_chol_solve(w->H, grad, nv, nbe, lane);
    real Ms = mw_matvec(w->M, w, search, nv, lane);
    if (lane < nv) w->vTmp[lane] = search;
    SYNCW();
    mw_J_times<SP>(w, w->eJv, w->sp->eJv, nefc, nv, lane);
    SYNCW();
    // exact line search (safeguarded Newton on a convex C1 function)
    real c1 = warp_sum(search * (Ma - qfs)), c2 = warp_sum(search * Ms);
    real cc, g1, g2;
    mw_linesearch_eval<SP>(w, lane, 0, &cc, &g1, &g2);
    real p1 = c1 + g1, p2 = c2 + g2;
    if (!(p1 < 0)) break;
    const real p10 = p1;
    real lo = 0, hi = -1, alpha = -p1 / p2;
    const real lstol = sizeof(real) == 4 ? (real)1e-5 : (real)1e-12;
    for (int ls = 0; ls < 24; ls++) {
      mw_linesearch_eval<SP>(w, lane, alpha, &cc, &g1, &g2);
      p1 = c1 + alpha * c2 + g1; p2 = c2 + g2;
      if (fabs(p1) < lstol * fabs(p10)) break;
      if (p1 < 0) lo = alpha; else hi = alpha;
      real an = alpha - p1 / p2;
      if (hi > 0 && (an <= lo || an >= hi)) an = (real)0.5 * (lo + hi);
      else if (hi < 0 && an <= lo) an = 2 * alpha;
      if (an == alpha) break;
      alpha = an;
    }
    qacc += alpha * search; Ma += alpha * Ms;
    for (int r = lane; r < nefc; r += 32) EV(eJar, r) += alpha * EV(eJv, r);
    SYNCW();
    real gauss = warp_sum((real)0.5 * (qacc - a0) * (Ma - qfs));
    real newcost = gauss + mw_constraint_eval<SP>(w, lane, false);
    SYNCW();
    real improvement = scale * (cost - newcost);
    cost = newcost;
    if (improvement < tol) { iter++; break; }
  }
  // (eF / fn are current: every exit from the loop follows an evaluation at the final point)
  real fc = 0;
  if (lane < nv) { for (int r = 0; r < nefc; r++) fc += JROW(r)[lane] * EV(eF, r); w->qacc[lane] = qacc; w->qfrc_con[lane] = fc; }
  if (lane == 0) w->solver_iter = iter;
  SYNCW();
}

// ------------------------------------------------------------------ forward dynamics + Euler
// mj_forward  (positions -> qacc); leaves link poses / contacts / efc forces in the scratch.
// PHASE_SYNC: the step kernel is far larger than the instruction cache, and with warps of one CTA spread over different phases
// most issue slots are lost to instruction fetch (ncu: stall_no_inst 55-60 %).  All warps of a CTA run the same model and make
// the same number of forward passes, so a CTA barrier at every phase boundary is legal; it keeps the CTA's warps inside the
// same code region and lets them share the fetched lines.  (Warps that have exited are not counted by the barrier.)
#define PHASE_SYNC() __syncthreads()
// which of the six phase boundaries of a forward pass carry a CTA barrier (bit i = boundary i: 0 entry, 1 after kinematics +
// inertia, 2 after collision, 3 after constraint rows, 4 after bias forces, 5 after the solver); tuned by measurement
#ifndef MW_SYNC_MASK
#define MW_SYNC_MASK 0x3f
#endif
#define PHASE_SYNC_AT(i) do { if (MW_SYNC_MASK & (1 << (i))) __syncthreads(); } while (0)
__device__ __noinline__ void mw_forward(const MwModel* __restrict__ m, const float* __restrict__ meshvert, WarpScratch* w, int lane) {
  const int nv = m->nv;
  long long t0 = MW_CLK(w), t1;
  PHASE_SYNC_AT(0);
  t1 = MW_CLK(w); if (lane == 0) w->prof[12] += t1 - t0; t0 = t1;
  // own work goes to prof[i]; the time spent waiting for the CTA's other warps at the phase boundary goes to prof[12]
#define PROF_(i, b) { t1 = MW_CLK(w); if (lane == 0) w->prof[i] += t1 - t0; PHASE_SYNC_AT(b); t0 = MW_CLK(w); if (lane == 0) w->prof[12] += t0 - t1; }
  mw_kinematics(m, w, lane);
  LaneDof L; mw_lane_dof(m, w, lane, &L);
  mw_mass_matrix(m, w, L, lane);
  PROF_(0, 1)
  mw_collide(m, meshvert, w, lane);
  PROF_(1, 2)
  const bool spill = w->ncon > MW_SMCON;          // this pass overflowed the shared-memory capacity (warp-uniform, rare)
  if (spill) mw_make_constraints<true>(m, w, L, lane); else mw_make_constraints<false>(m, w, L, lane);
  PROF_(3, 3)
  real bias = mw_rne_bias(m, w, L, lane);
  // passive + actuation  [mj_passive, mj_fwdActuation]
  real qfs = 0;
  if (L.valid) {
    real qv = w->qvel[lane];
    qfs = -m->dof_damping[lane] * qv - bias;
    real k = m->dof_stiffness[lane];
    if (k != 0) qfs -= k * (w->qpos[m->dof_qadr[lane]] - m->dof_springref[lane]);
    for (int u = 0; u < 2; u++) if (m->act_dof[u] == lane) {
      real c = fmin(fmax(w->ctrl[u], (real)m->act_lo[u]), (real)m->act_hi[u]);
      qfs += m->act_kp[u] * (c - w->qpos[m->dof_qadr[lane]]);
    }
    w->qfrc_smooth[lane] = qfs;
  }
  // qacc_smooth = M^-1 qfrc_smooth (factor in H)
  for (int i = lane; i < nv * NVP; i += 32) w->H[i] = w->M[i];
  SYNCW();
  const int nbe = mw_chol(w->H, nv, w->nblk1, lane);
  real as = mw_chol_solve(w->H, qfs, nv, nbe, lane);
  if (lane < nv) w->qacc_smooth[lane] = as;
  SYNCW();
  PROF_(4, 4)
  if (spill) mw_solve<true>(m, w, lane, sizeof(real) == 4 ? 8 : 50); else mw_solve<false>(m, w, lane, sizeof(real) == 4 ? 8 : 50);
  PROF_(5, 5)
#undef PROF_
}

// positions only: what the last mj_forward of an env step contributes when nothing reads its contacts / forces
// (same CTA barrier as the start of mw_forward, so the warps of a CTA stay phase-aligned)
__device__ __noinline__ void mw_forward_kinematics_only(const MwModel* __restrict__ m, WarpScratch* w, int lane) {
  long long t0 = MW_CLK(w), t1;
  PHASE_SYNC_AT(0);
  t1 = MW_CLK(w); if (lane == 0) w->prof[12] += t1 - t0; t0 = t1;
  mw_kinematics(m, w, lane);
  t1 = MW_CLK(w); if (lane == 0) w->prof[0] += t1 - t0;
  if (lane == 0) { w->solver_iter = 0; w->ncon_dropped = 0; }
  SYNCW();
}

// mj_Euler: semi-implicit, joint damping implicit
__device__ __noinline__ void mw_euler(const MwModel* __restrict__ m, WarpScratch* w, int lane) {
  const int nv = m->nv; const real h = m->timestep;
  for (int i = lane; i < nv * NVP; i += 32) w->H[i] = w->M[i];
  SYNCW();
  if (lane < nv) w->H[lane * NVP + lane] += h * m->dof_damping[lane];
  SYNCW();
  const int nbe = mw_chol(w->H, nv, w->nblk1, lane);
  real rhs = lane < nv ? w->qfrc_smooth[lane] + w->qfrc_con[lane] : (real)0;
  real acc = mw_chol_solve(w->H, rhs, nv, nbe, lane);
  if (lane < nv) { w->qvel[lane] += h * acc; w->warm[lane] = w->qacc[lane]; }
  SYNCW();
  // positions (float64 state; the float copy is refreshed for the dynamics)
  if (lane < m->nlink) {
    int l = lane, jt = m->link_jtype[l], qa = m->link_qadr[l], da = m->link_dadr[l];
    const double hd = (double)h;
    if (jt == JT_FREE) {
      for (int i = 0; i < 3; i++) QSET(w, qa + i, w->qposd[qa + i] + hd * (double)w->qvel[da + i]);
      double wv[3] = {w->qvel[da + 3], w->qvel[da + 4], w->qvel[da + 5]};
      double n = v3norm(wv);
      if (n >= (double)MW_EPS) {
        double ax[3] = {wv[0] / n, wv[1] / n, wv[2] / n}, dq[4], q[4] = {w->qposd[qa + 3], w->qposd[qa + 4], w->qposd[qa + 5], w->qposd[qa + 6]}, r[4];
        quat_axisangle(dq, ax, n * hd);
        quat_mul(r, q, dq); quat_normalize(r);
        for (int i = 0; i < 4; i++) QSET(w, qa + 3 + i, r[i]);
      }
    } else QSET(w, qa, w->qposd[qa] + hd * (double)w->qvel[da]);
  }
  SYNCW();
}
