// Host emulation of the device kinematics and bias forces (mw_kinematics, mw_link_inertia, mw_rne_bias in
// metaworld_b200/csrc/mw_physics.cuh) with a full warp: the CUDA source is compiled by g++ and run as 32 cooperative
// fibers, one per lane, that hand over to the next lane at every __syncwarp().  Between two __syncwarp() points a lane
// therefore sees exactly the shared-memory writes a real warp guarantees it: those made before the previous barrier.
// Built twice by tests/test_kinematics_lanes.py, with and without -DMW_SERIAL_LINKS; the two libraries must write the
// same bytes.  The functions under test use no shuffles; the stubs below only let the rest of the header compile.
// Test infrastructure only.
#define MW_HOST_EMU
#define MW_WARP 32
#include <cmath>
#include <cstring>
#include <ucontext.h>
#define __device__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
template <class T> static inline T __shfl_sync(unsigned, T v, int) { return v; }
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int) { return v; }
template <class T> static inline T __shfl_up_sync(unsigned, T v, int) { return v; }
static inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }
static inline bool __any_sync(unsigned, bool p) { return p; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
static inline int atomicAdd(int* p, int v) { int o = *p; *p += v; return o; }
static inline void __syncthreads() {}
static struct { int x; } threadIdx;
template <class T> static inline T __ldg(const T* p) { return *p; }
struct float4 { float x, y, z, w; };

static ucontext_t g_main, g_lane[32];
static int g_cur;
static volatile int g_yielded;
static void __syncwarp() { g_yielded = 1; swapcontext(&g_lane[g_cur], &g_main); }

#include "../../metaworld_b200/csrc/mw_physics.cuh"

static WarpScratch g_w;
static const MwModel* g_m;
static real g_bias[32];
static char g_stack[32][1 << 16];

static void lane_main(int lane) {
  mw_kinematics(g_m, &g_w, lane);
  LaneDof L; mw_lane_dof(g_m, &g_w, lane, &L);
  mw_link_inertia(g_m, &g_w, lane);
  g_bias[lane] = mw_rne_bias(g_m, &g_w, L, lane);
}

template <class T> static char* put(char* o, const T& x) { memcpy(o, &x, sizeof(T)); return o + sizeof(T); }

// One pass for one env: positions `qposd` [MW_MAXNQ], velocities `qvel` [MW_MAXDOF], world shift [3].  Writes the link
// poses, dof axes and anchors, the written-back positions and the 32 lanes' bias forces to `out`; returns the byte count.
extern "C" int kin_pass(const void* model, const double* qposd, const double* qvel, const double* shift, char* out) {
  g_m = (const MwModel*)model;
  memset(&g_w, 0, sizeof(g_w));
  for (int i = 0; i < MW_MAXNQ; i++) { g_w.qposd[i] = qposd[i]; g_w.qpos[i] = (real)qposd[i]; }
  for (int i = 0; i < MW_MAXDOF; i++) g_w.qvel[i] = (real)qvel[i];
  for (int i = 0; i < 3; i++) g_w.shift[i] = (real)shift[i];
  bool done[32];
  for (int l = 0; l < 32; l++) {
    getcontext(&g_lane[l]);
    g_lane[l].uc_stack.ss_sp = g_stack[l]; g_lane[l].uc_stack.ss_size = sizeof(g_stack[l]);
    g_lane[l].uc_link = &g_main;
    makecontext(&g_lane[l], (void (*)())lane_main, 1, l);
    done[l] = false;
  }
  // a lane comes back here either from __syncwarp() or, through uc_link, when lane_main returned; every lane meets the
  // same number of barriers, so all of them finish in the same round
  for (int live = 32; live > 0;) {
    for (int l = 0; l < 32; l++) if (!done[l]) {
      g_cur = l; g_yielded = 0;
      swapcontext(&g_main, &g_lane[l]);
      if (!g_yielded) { done[l] = true; live--; }
    }
  }
  char* o = out;
  o = put(o, g_w.lposd); o = put(o, g_w.lquatd); o = put(o, g_w.lpos); o = put(o, g_w.lquat); o = put(o, g_w.lmat);
  o = put(o, g_w.daxis); o = put(o, g_w.danchor); o = put(o, g_w.qposd); o = put(o, g_w.qpos); o = put(o, g_bias);
  return (int)(o - out);
}
