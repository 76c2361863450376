// The 50 scripted expert policies of metaworld.policies (ENV_POLICY_MAP, metaworld/policies/__init__.py:76), restated by
// hand: one pure function obs[:39] -> action[4] per task, selected by the task ids of mw_task_ids.h.
//
// Arithmetic follows the reference's numpy float64 path exactly: the observation is widened to double, every vector
// offset is added component by component (including the zero ones, so signed zeros come out as numpy's do),
// np.linalg.norm is the square root of the in-order sum of squares, and move() is p * (target - hand), rounded to float32
// once at the end (Action.array is float32).  Nothing is clipped: the reference returns unclipped actions and the step
// clips them.  Only + - * / sqrt fabs and comparisons are used; with contraction off (nvcc --fmad=false, g++
// -ffp-contract=off) the device and host builds of this header give identical bits.
//
// Compiles under nvcc and under a plain C++ compiler (tests/devpolicy/shim.cpp): no warp intrinsics, no device-only calls.
#pragma once
#include <math.h>

#include "mw_task_ids.h"

#ifndef MWP_DEV
#ifdef __CUDACC__
#define MWP_DEV __host__ __device__ __forceinline__
#else
#define MWP_DEV static inline
#endif
#endif

struct PV { double x, y, z; };

MWP_DEV PV pv(double x, double y, double z) { PV r; r.x = x; r.y = y; r.z = z; return r; }
MWP_DEV PV pv_add(PV a, double x, double y, double z) { return pv(a.x + x, a.y + y, a.z + z); }
// np.linalg.norm of the xy / xz / yz / xyz difference
MWP_DEV double pv_dxy(PV a, PV b) { double u = a.x - b.x, v = a.y - b.y; return sqrt(u * u + v * v); }
MWP_DEV double pv_dxz(PV a, PV b) { double u = a.x - b.x, v = a.z - b.z; return sqrt(u * u + v * v); }
MWP_DEV double pv_dyz(PV a, PV b) { double u = a.y - b.y, v = a.z - b.z; return sqrt(u * u + v * v); }
MWP_DEV double pv_d3(PV a, PV b) { double u = a.x - b.x, v = a.y - b.y, w = a.z - b.z; return sqrt(u * u + v * v + w * w); }
// np.isclose(x, y, atol=atol) with the default rtol: (|x - y| <= atol + rtol |y| and y finite) or x == y
MWP_DEV bool pv_isclose(double x, double y, double atol) {
  return (fabs(x - y) <= atol + 1e-05 * fabs(y) && y - y == 0.0) || x == y;
}
// the stick tasks: the two-stage approach to the stick, then to the thermos (the same decision tree, different offsets)
MWP_DEV PV pv_stick(PV hand, PV stick, PV thermos, PV goal) {
  if (fabs(stick.x - thermos.x) > 0.04) {
    if (pv_dxy(hand, stick) > 0.02) return pv_add(stick, 0.0, 0.0, 0.1);
    if (fabs(hand.z - stick.z) > 0.02) return stick;
    if (fabs(stick.y - thermos.y) > 0.02) return pv(stick.x, thermos.y, stick.z);
    if (fabs(stick.z - thermos.z) > 0.02) return pv(stick.x, thermos.y, thermos.z);
    return thermos;
  }
  return goal;
}

// a[0:3] = move(hand, target, p), a[3] = the grab effort.  An id outside [0, T_NTASK) gives a NaN row.
MWP_DEV void policy_action(int task_id, const double o[39], float a[4]) {
  const PV hand = pv(o[0], o[1], o[2]), obj = pv(o[4], o[5], o[6]), goal = pv(o[36], o[37], o[38]);
  PV to = hand;
  double p = 25.0, grab = 0.0;
  switch (task_id) {
    case T_ASSEMBLY: {                       // sawyer_assembly_v3_policy.py:24-69
      p = 10.0;
      const PV w = pv_add(obj, -0.02, 0.0, 0.0), peg = pv_add(goal, 0.12, 0.0, 0.14);
      if (pv_dxy(hand, w) > 0.02) to = pv_add(w, 0.0, 0.0, 0.1);
      else if (pv_dxy(hand, peg) <= 0.02) to = pv_add(peg, 0.0, 0.0, -0.2);
      else if (fabs(hand.z - w.z) > 0.05) to = pv_add(w, 0.0, 0.0, 0.03);
      else if (fabs(hand.z - peg.z) > 0.04) to = pv(hand.x, hand.y, peg.z);
      else to = peg;
      grab = (pv_dxy(hand, w) > 0.02 || fabs(hand.z - w.z) > 0.12) ? 0.0 : 0.6;
    } break;
    case T_BASKETBALL: {                     // sawyer_basketball_v3_policy.py:25-62
      const PV ball = pv_add(obj, 0.0, 0.0, 0.01), hoop = pv(o[36], 0.875, 0.35);
      if (pv_dxy(hand, ball) > 0.04) to = pv_add(ball, 0.0, 0.0, 0.3);
      else if (fabs(hand.z - ball.z) > 0.025) to = ball;
      else if (fabs(ball.z - hoop.z) > 0.025) to = pv(hand.x, hand.y, hoop.z);
      else to = hoop;
      grab = (pv_dxy(hand, obj) > 0.04 || fabs(hand.z - obj.z) > 0.15) ? -1.0 : 0.6;
    } break;
    case T_BIN_PICKING: {                    // sawyer_bin_picking_v3_policy.py:23-72
      PV cube = pv_add(obj, 0.0, 0.0, 0.03);
      double cy = (0.725 < cube.y) ? 0.725 : cube.y;        // Python's max(0.675, min(y, 0.725))
      cube.y = (cy > 0.675) ? cy : 0.675;
      const PV bin = pv(0.12, 0.7, 0.02);
      if (pv_dxy(hand, cube) > 0.02) to = pv_add(cube, 0.0, 0.0, 0.15);
      else if (fabs(hand.z - cube.z) > 0.01) to = cube;
      else if (pv_dxy(hand, bin) > 0.02) to = hand.z < 0.15 ? pv_add(hand, 0.0, 0.0, 0.1) : pv(bin.x, bin.y, 0.18);
      else to = bin;
      grab = (pv_dxy(hand, cube) > 0.02 || fabs(hand.z - cube.z) > 0.02) ? -1.0 : 0.6;
    } break;
    case T_BOX_CLOSE: {                      // sawyer_box_close_v3_policy.py:25-67
      const PV lid = pv_add(obj, 0.0, 0.0, 0.02), box = pv_add(pv(o[36], o[37], 0.15), 0.0, 0.0, 0.0);
      if (pv_dxy(hand, lid) > 0.01) to = pv(lid.x, lid.y, 0.2);
      else if (fabs(hand.z - lid.z) > 0.05) to = lid;
      else if (fabs(hand.z - box.z) > 0.04) to = pv(hand.x, hand.y, box.z);
      else to = box;
      grab = (pv_dxy(hand, lid) > 0.01 || fabs(hand.z - lid.z) > 0.13) ? 0.5 : 1.0;
    } break;
    case T_BUTTON_PRESS_TOPDOWN:             // sawyer_button_press_topdown_v3_policy.py:23-43
      to = pv_dxy(hand, obj) > 0.04 ? pv_add(obj, 0.0, 0.0, 0.1) : obj;
      grab = 1.0;
      break;
    case T_BUTTON_PRESS_TOPDOWN_WALL: {      // sawyer_button_press_topdown_wall_v3_policy.py:23-43
      const PV b = pv_add(obj, 0.0, -0.06, 0.0);
      to = pv_dxy(hand, b) > 0.04 ? pv_add(b, 0.0, 0.0, 0.1) : b;
      grab = -1.0;
    } break;
    case T_BUTTON_PRESS: {                   // sawyer_button_press_v3_policy.py:22-56
      PV b = pv_add(obj, 0.0, 0.0, -0.07);
      if (!(pv_isclose(hand.x, b.x, 0.02) && pv_isclose(hand.z, b.z, 0.02))) b.y = hand.y - 0.1;
      else b.y += 0.02;
      to = b;
      grab = 0.0;
    } break;
    case T_BUTTON_PRESS_WALL: {              // sawyer_button_press_wall_v3_policy.py:22-60
      p = 15.0;
      const PV b = pv_add(obj, 0.0, 0.0, 0.04);
      const bool far_x = fabs(hand.x - b.x) > 0.02, far_y = b.y - hand.y > 0.09, far_z = fabs(hand.z - b.z) > 0.02;
      if (far_x) to = pv(b.x, hand.y, 0.3);
      else if (far_y) to = pv(b.x, b.y, 0.3);
      else if (far_z) to = pv_add(b, 0.0, -0.05, 0.0);
      else to = pv_add(b, 0.0, -0.02, 0.0);
      grab = (far_x || far_y || far_z) ? 1.0 : -1.0;
    } break;
    case T_COFFEE_BUTTON: {                  // sawyer_coffee_button_v3_policy.py:23-43
      p = 10.0;
      const PV b = pv_add(obj, 0.0, 0.0, -0.07);
      to = pv_dxz(hand, b) > 0.02 ? pv(b.x, hand.y, b.z) : pv_add(b, 0.0, 0.2, 0.0);
      grab = -1.0;
    } break;
    case T_COFFEE_PULL: {                    // sawyer_coffee_pull_v3_policy.py:24-59
      p = 10.0;
      const PV mug = pv_add(obj, -0.005, 0.0, 0.05), mug_g = pv_add(obj, 0.01, 0.0, 0.05);
      if (pv_dxy(hand, mug) > 0.06) to = pv_add(mug, 0.0, 0.0, 0.15);
      else if (fabs(hand.z - mug.z) > 0.02) to = mug;
      else to = goal;
      grab = (pv_dxy(hand, mug_g) > 0.06 || fabs(hand.z - mug_g.z) > 0.1) ? -1.0 : 0.7;
    } break;
    case T_COFFEE_PUSH: {                    // sawyer_coffee_push_v3_policy.py:25-61
      p = 10.0;
      const PV mug = pv_add(obj, 0.01, 0.0, 0.05);
      if (pv_dxy(hand, mug) > 0.06) to = pv_add(mug, 0.0, 0.0, 0.2);
      else if (fabs(hand.z - mug.z) > 0.02) to = mug;
      else to = pv(o[36], o[37], 0.1);
      grab = (pv_dxy(hand, mug) > 0.06 || fabs(hand.z - mug.z) > 0.1) ? -1.0 : 0.5;
    } break;
    case T_DIAL_TURN: {                      // sawyer_dial_turn_v3_policy.py:23-44
      p = 10.0;
      const PV d = pv_add(obj, 0.05, 0.02, 0.09);
      if (pv_dxy(hand, d) > 0.02) to = pv(d.x, d.y, 0.2);
      else if (fabs(hand.z - d.z) > 0.02) to = d;
      else to = pv_add(d, -0.05, 0.005, 0.0);
      grab = 1.0;
    } break;
    case T_DISASSEMBLE: {                    // sawyer_disassemble_v3_policy.py:24-63
      p = 10.0;
      const PV w = pv_add(obj, -0.02, 0.0, 0.01);
      if (pv_dxy(hand, w) > 0.02) to = pv_add(w, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - w.z) > 0.03) to = w;
      else to = pv_add(hand, 0.0, 0.0, 0.1);
      grab = (pv_dxy(hand, w) > 0.02 || fabs(hand.z - w.z) > 0.07) ? 0.0 : 0.8;
    } break;
    case T_DOOR_CLOSE: {                     // sawyer_door_close_v3_policy.py:24-57
      const PV d = pv_add(obj, 0.05, 0.12, 0.1);
      if (hand.x > d.x) to = hand.z < d.z + 0.2 ? pv(hand.x, hand.y, d.z + 0.25) : pv(d.x - 0.02, d.y, hand.z);
      else if (fabs(hand.z - d.z) > 0.04) to = pv_add(d, -0.02, 0.0, 0.0);
      else to = goal;
      grab = 1.0;
    } break;
    case T_DOOR_LOCK: {                      // sawyer_door_lock_v3_policy.py:23-47
      const PV l = pv_add(obj, -0.02, -0.02, 0.0);
      if (pv_dxy(hand, l) > 0.02) to = hand.z < 0.25 ? pv_add(hand, 0.0, -0.1, 0.1) : pv_add(l, 0.0, 0.0, 0.3);
      else if (fabs(hand.z - l.z) > 0.02) to = l;
      else to = pv_add(l, -0.1, 0.0, -0.1);
      grab = -1.0;
    } break;
    case T_DOOR_OPEN: {                      // sawyer_door_open_v3_policy.py:23-49
      const PV d = pv(obj.x - 0.05, obj.y, obj.z);
      if (pv_dxy(hand, d) > 0.12) to = pv_add(d, 0.06, 0.02, 0.2);
      else if (fabs(hand.z - d.z) > 0.04) to = pv_add(d, 0.06, 0.02, 0.0);
      else to = d;
      grab = 1.0;
    } break;
    case T_DOOR_UNLOCK: {                    // sawyer_door_unlock_v3_policy.py:23-45
      const PV l = pv_add(obj, -0.04, -0.02, -0.03);
      if (pv_dxy(hand, l) > 0.02) to = hand.z > 0.15 ? pv_add(hand, 0.0, -0.1, -0.1) : l;
      else to = pv_add(l, 0.1, 0.0, 0.01);
      grab = 1.0;
    } break;
    case T_DRAWER_CLOSE: {                   // sawyer_drawer_close_v3_policy.py:23-53
      const PV d = pv_add(obj, 0.0, 0.0, -0.02);
      if (hand.y > d.y) to = hand.z < d.z + 0.23 ? pv(hand.x, hand.y, d.z + 0.5) : pv_add(d, 0.0, -0.075, 0.23);
      else if (fabs(hand.z - d.z) > 0.04) to = pv_add(d, 0.0, -0.075, 0.0);
      else to = d;
      grab = 1.0;
    } break;
    case T_DRAWER_OPEN: {                    // sawyer_drawer_open_v3_policy.py:21-48
      const PV d = pv_add(obj, 0.0, 0.0, -0.02);
      if (pv_dxy(hand, d) > 0.06) { to = pv_add(d, 0.0, 0.0, 0.3); p = 4.0; }
      else if (fabs(hand.z - d.z) > 0.04) { to = d; p = 4.0; }
      else { to = pv_add(d, 0.0, -0.06, 0.0); p = 50.0; }
      grab = -1.0;
    } break;
    case T_FAUCET_CLOSE: {                   // sawyer_faucet_close_v3_policy.py:23-45
      const PV f = pv_add(obj, 0.04, 0.0, 0.03);
      if (pv_dxy(hand, f) > 0.04) to = pv_add(f, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - f.z) > 0.04) to = f;
      else to = pv_add(f, -0.1, 0.05, 0.0);
      grab = 1.0;
    } break;
    case T_FAUCET_OPEN: {                    // sawyer_faucet_open_v3_policy.py:23-45
      const PV f = pv_add(obj, -0.04, 0.0, 0.03);
      if (pv_dxy(hand, f) > 0.04) to = pv_add(f, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - f.z) > 0.04) to = f;
      else to = pv_add(f, 0.1, 0.05, 0.0);
      grab = 1.0;
    } break;
    case T_HAMMER: {                         // sawyer_hammer_v3_policy.py:23-65
      p = 10.0;
      const PV h = pv_add(obj, -0.04, 0.0, -0.01), g = pv_add(pv(0.24, 0.71, 0.11), -0.19, 0.0, 0.05);
      if (pv_dxy(hand, h) > 0.04) to = pv_add(h, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - h.z) > 0.05 && h.z < 0.03) to = pv_add(h, 0.0, 0.0, 0.03);
      else if (pv_dxz(hand, g) > 0.02) to = pv(g.x, hand.y, g.z);
      else to = g;
      grab = (pv_dxy(hand, h) > 0.04 || fabs(hand.z - h.z) > 0.1) ? 0.0 : 0.8;
    } break;
    case T_HAND_INSERT:                      // sawyer_hand_insert_v3_policy.py:24-64
      p = 10.0;
      if (pv_dxy(hand, obj) > 0.02) to = pv_add(obj, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - obj.z) > 0.05) to = pv_add(obj, 0.0, 0.0, 0.03);
      else if (pv_dxy(hand, goal) > 0.04) to = pv(goal.x, goal.y, hand.z);
      else to = goal;
      grab = (pv_dxy(hand, obj) > 0.02 || fabs(hand.z - obj.z) > 0.1) ? 0.0 : 0.65;
      break;
    case T_HANDLE_PRESS_SIDE:                // sawyer_handle_press_side_v3_policy.py:23-43
      to = pv_dxy(hand, obj) > 0.02 ? pv_add(obj, 0.0, 0.0, 0.2) : pv_add(obj, 0.0, 0.0, -0.5);
      grab = 1.0;
      break;
    case T_HANDLE_PRESS: {                   // sawyer_handle_press_v3_policy.py:23-43
      const PV b = pv_add(obj, 0.0, -0.02, 0.0);
      to = pv_dxy(hand, b) > 0.02 ? pv_add(b, 0.0, 0.0, 0.2) : pv_add(b, 0.0, 0.0, -0.5);
      grab = -1.0;
    } break;
    case T_HANDLE_PULL_SIDE:                 // sawyer_handle_pull_side_v3_policy.py:22-54
      if (pv_dxy(hand, obj) > 0.04) to = pv_add(obj, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - obj.z) > 0.03) to = obj;
      else to = pv_add(obj, 0.0, 0.0, 1.0);
      grab = (pv_dxy(hand, obj) > 0.04 || fabs(hand.z - obj.z) > 0.04) ? 0.0 : 0.6;
      break;
    case T_HANDLE_PULL: {                    // sawyer_handle_pull_v3_policy.py:22-47
      const PV h = pv_add(obj, 0.0, -0.04, 0.0);
      if (pv_dxy(hand, h) > 0.02) to = h;
      else if (fabs(hand.z - h.z) > 0.02) to = pv(h.z, h.z, h.z);    // the reference returns the scalar z: move() broadcasts it
      else to = pv_add(h, 0.0, 0.0, 0.1);
      grab = 1.0;
    } break;
    case T_LEVER_PULL: {                     // sawyer_lever_pull_v3_policy.py:23-45
      const PV l = pv_add(obj, 0.0, -0.055, 0.0);
      if (pv_dxy(hand, l) > 0.02) to = pv_add(l, 0.0, 0.0, -0.1);
      else if (fabs(hand.z - l.z) > 0.02) to = l;
      else to = pv_add(l, 0.0, 0.08, 0.02);
      grab = 1.0;
    } break;
    case T_PEG_INSERT_SIDE: {                // sawyer_peg_insertion_side_v3_policy.py:26-67
      const PV hole = pv(-0.35, o[37], 0.16);
      if (pv_dxy(hand, obj) > 0.04) to = pv_add(obj, 0.0, 0.0, 0.3);
      else if (fabs(hand.z - obj.z) > 0.025) to = obj;
      else if (pv_dyz(obj, hole) > 0.03) to = pv_add(hole, 0.4, 0.0, 0.0);
      else to = hole;
      grab = (pv_dxy(hand, obj) > 0.04 || fabs(hand.z - obj.z) > 0.15) ? -1.0 : 0.6;
    } break;
    case T_PEG_UNPLUG_SIDE: {                // sawyer_peg_unplug_side_v3_policy.py:23-58
      const PV peg = pv_add(obj, -0.02, 0.0, 0.035);
      if (pv_dxy(hand, peg) > 0.04) to = pv_add(peg, 0.0, 0.0, 0.2);
      else if (fabs(hand.z - 0.15) > 0.02) to = pv(peg.x, peg.y, 0.15);
      else to = pv_add(hand, 0.01, 0.0, 0.0);
      grab = (pv_dxy(hand, peg) > 0.04 || fabs(hand.z - peg.z) > 0.15) ? -1.0 : 0.1;
    } break;
    case T_PICK_OUT_OF_HOLE: {               // sawyer_pick_out_of_hole_v3_policy.py:24-67
      const PV puck = pv_add(obj, 0.0, 0.0, 0.02);
      if (pv_dxy(hand, puck) > 0.02) to = pv_add(puck, 0.0, 0.0, 0.15);
      else if (fabs(hand.z - puck.z) > 0.01) to = puck;
      else if (fabs(hand.z - goal.z) > 0.04) to = pv(hand.x, hand.y, goal.z);
      else to = goal;
      grab = (pv_dxy(hand, puck) > 0.02 || fabs(hand.z - puck.z) > 0.15) ? 0.0 : 0.1;
    } break;
    case T_PICK_PLACE: {                     // sawyer_pick_place_v3_policy.py:26-64
      p = 10.0;
      const PV puck = pv_add(obj, -0.005, 0.0, 0.0);
      if (pv_dxy(hand, puck) > 0.02) to = pv_add(puck, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - puck.z) > 0.05 && puck.z < 0.04) to = pv_add(puck, 0.0, 0.0, 0.03);
      else if (o[3] > 0.73) to = hand;
      else to = goal;
      grab = pv_d3(hand, obj) < 0.07 ? 1.0 : 0.0;
    } break;
    case T_PICK_PLACE_WALL: {                // sawyer_pick_place_wall_v3_policy.py:24-81
      p = 10.0;
      const PV puck = pv_add(obj, -0.005, 0.0, 0.0);
      const bool over_wall = -0.15 <= hand.x && hand.x <= 0.35 && 0.6 <= hand.y && hand.y <= 0.8;
      if (pv_dxy(hand, puck) > 0.015) to = pv_add(puck, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - puck.z) > 0.04 && puck.z < 0.03) to = pv_add(puck, 0.0, 0.0, 0.03);
      else if (over_wall && hand.z < 0.25) to = pv_add(hand, 0.0, 0.0, 1.0);
      else if (over_wall && hand.z < 0.35) to = pv(goal.x, goal.y, hand.z);
      else if (fabs(hand.z - goal.z) > 0.01) to = pv(hand.x, hand.y, goal.z);
      else to = goal;
      grab = (pv_dxy(hand, obj) > 0.015 || fabs(hand.z - obj.z) > 0.1) ? 0.0 : 0.9;
    } break;
    case T_PLATE_SLIDE_BACK_SIDE: {          // sawyer_plate_slide_back_side_v3_policy.py:23-45
      p = 10.0;
      const PV puck = pv_add(obj, 0.023, 0.0, 0.025);
      if (pv_dxy(hand, puck) > 0.01) to = pv_add(puck, 0.0, 0.0, 0.07);
      else if (fabs(hand.z - puck.z) > 0.04) to = puck;
      else to = pv(hand.x + 0.1, 0.6, hand.z);
      grab = 1.0;
    } break;
    case T_PLATE_SLIDE_BACK: {               // sawyer_plate_slide_back_v3_policy.py:23-49
      p = 10.0;
      const PV puck = pv_add(obj, 0.0, -0.065, 0.025);
      if (pv_dxy(hand, puck) > 0.01) to = pv_add(puck, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - puck.z) > 0.04) to = puck;
      else if (hand.y > 0.7) to = pv_add(hand, 0.0, -0.1, 0.0);
      else if (hand.y > 0.6) to = pv(0.15, 0.55, hand.z);
      else to = pv(hand.x - 0.1, 0.55, hand.z);
      grab = -1.0;
    } break;
    case T_PLATE_SLIDE_SIDE: {               // sawyer_plate_slide_side_v3_policy.py:28-52
      const PV puck = pv_add(obj, 0.07, 0.0, -0.005);
      if (pv_dxy(hand, puck) > 0.04) to = pv_add(puck, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - puck.z) > 0.04) to = puck;
      else if (hand.x > -0.2) to = pv(hand.x - 0.1, 0.6, hand.z);
      else to = pv_add(puck, -0.1, 0.0, 0.0);
      grab = 1.0;
    } break;
    case T_PLATE_SLIDE: {                    // sawyer_plate_slide_v3_policy.py:25-49
      p = 10.0;
      const PV puck = pv_add(obj, 0.0, -0.055, 0.03);
      if (!(pv_dxy(hand, puck) <= 0.03)) to = pv_add(puck, 0.0, 0.0, 0.1);
      else if (fabs(hand.z - puck.z) > 0.04) to = puck;
      else to = pv(o[36], 0.9, puck.z);
      grab = -1.0;
    } break;
    case T_PUSH_BACK:                        // sawyer_push_back_v3_policy.py:24-63
      p = 10.0;
      if (pv_dxy(hand, obj) > 0.04) to = pv_add(obj, 0.0, 0.0, 0.3);
      else if (fabs(hand.z - obj.z) > 0.055) to = obj;
      else to = pv_add(goal, 0.0, 0.0, hand.z);
      grab = (pv_dxy(hand, obj) > 0.04 || fabs(hand.z - obj.z) > 0.05) ? 0.0 : 0.9;
      break;
    case T_PUSH: {                           // sawyer_push_v3_policy.py:24-64
      p = 10.0;
      const PV puck = pv_add(obj, -0.005, 0.0, 0.0);
      if (pv_dxy(hand, puck) > 0.02) to = pv_add(puck, 0.0, 0.0, 0.2);
      else if (fabs(hand.z - puck.z) > 0.04) to = pv_add(puck, 0.0, 0.0, 0.03);
      else to = goal;
      grab = (pv_dxy(hand, obj) > 0.02 || fabs(hand.z - obj.z) > 0.1) ? 0.0 : 0.6;
    } break;
    case T_PUSH_WALL: {                      // sawyer_push_wall_v3_policy.py:24-69
      p = 10.0;
      const PV b = pv_add(obj, -0.005, 0.0, 0.0);
      if (pv_dxy(hand, b) > 0.02) to = pv_add(b, 0.0, 0.0, 0.2);
      else if (fabs(hand.z - b.z) > 0.04) to = pv_add(b, 0.0, 0.0, 0.03);
      else if (-0.1 <= b.x && b.x <= 0.3 && 0.65 <= b.y && b.y <= 0.75) to = pv_add(hand, -1.0, 0.0, 0.0);
      else if (((-0.15 < b.x && b.x < 0.05) || (0.15 < b.x && b.x < 0.35)) && 0.695 <= b.y && b.y <= 0.755) to = pv_add(hand, 0.0, 1.0, 0.0);
      else to = goal;
      grab = (pv_dxy(hand, obj) > 0.02 || fabs(hand.z - obj.z) > 0.1) ? 0.0 : 0.6;
    } break;
    case T_REACH:                            // sawyer_reach_v3_policy.py:22-30
      p = 5.0;
      to = goal;
      grab = 0.0;
      break;
    case T_REACH_WALL:                       // sawyer_reach_wall_v3_policy.py:23-47
      p = 5.0;
      to = (-0.1 <= hand.x && hand.x <= 0.3 && 0.6 <= hand.y && hand.y <= 0.8 && hand.z < 0.25) ? pv_add(goal, 0.0, 0.0, 1.0) : goal;
      grab = 0.0;
      break;
    case T_SHELF_PLACE: {                    // sawyer_shelf_place_v3_policy.py:25-71
      const PV blk = pv_add(obj, -0.005, 0.0, 0.015);
      const double shelf_x = o[36];
      if (pv_dxy(hand, blk) > 0.04) to = pv_add(blk, 0.0, 0.0, 0.3);
      else if (fabs(hand.z - blk.z) > 0.04) to = blk;
      else if (fabs(hand.x - shelf_x) > 0.02) to = pv(shelf_x, hand.y, 0.3);
      else if (hand.z < 0.3) to = pv_add(hand, 0.0, 0.0, 0.3);
      else to = pv_add(hand, 0.0, 0.05, 0.0);
      grab = (pv_dxy(hand, obj) > 0.04 || fabs(hand.z - obj.z) > 0.15) ? -1.0 : 0.7;
    } break;
    case T_SOCCER: {                         // sawyer_soccer_v3_policy.py:24-58
      const PV ball = pv_add(obj, 0.0, 0.0, 0.03);
      const double want_z = pv_dxy(hand, ball) < 0.02 ? 0.1 : 0.03;
      PV push = pv_add(ball, 0.0, -0.03, 0.0);
      if (ball.x - goal.x < -0.05) push = pv_add(ball, -0.03, 0.0, 0.0);
      else if (ball.x - goal.x > 0.05) push = pv_add(ball, 0.03, 0.0, 0.0);
      push.z = want_z;
      to = pv_d3(hand, push) > 0.01 ? push : ball;
      grab = 1.0;
    } break;
    case T_STICK_PULL: {                     // sawyer_stick_pull_v3_policy.py:26-70
      const PV stick = pv_add(obj, -0.015, 0.0, 0.03);
      to = pv_stick(hand, stick, pv_add(pv(o[11], o[12], o[13]), -0.015, 0.0, 0.03), pv_add(goal, -0.05, 0.0, 0.0));
      grab = (pv_dxy(hand, stick) > 0.02 || fabs(hand.z - stick.z) > 0.1) ? -1.0 : 0.7;
    } break;
    case T_STICK_PUSH: {                     // sawyer_stick_push_v3_policy.py:26-70
      p = 10.0;
      const PV stick = pv_add(obj, 0.015, 0.0, 0.03);
      to = pv_stick(hand, stick, pv(o[11], o[12], o[13]), pv_add(goal, 0.0, 0.0, 0.132));
      grab = (pv_dxy(hand, stick) > 0.02 || fabs(hand.z - stick.z) > 0.1) ? -1.0 : 0.7;
    } break;
    case T_SWEEP_INTO: {                     // sawyer_sweep_into_v3_policy.py:24-60
      const PV cube = pv_add(obj, -0.005, 0.0, 0.01);
      if (pv_dxy(hand, cube) > 0.04) to = pv_add(cube, 0.0, 0.0, 0.3);
      else if (fabs(hand.z - cube.z) > 0.04) to = cube;
      else to = goal;
      grab = (pv_dxy(hand, obj) > 0.04 || fabs(hand.z - obj.z) > 0.15) ? -1.0 : 0.7;
    } break;
    case T_SWEEP: {                          // sawyer_sweep_v3_policy.py:24-63
      const PV cube = pv_add(obj, 0.0, 0.0, 0.015);
      if (hand.x < 0.2 && pv_dxy(hand, cube) > 0.04) to = pv_add(cube, 0.0, 0.0, 0.3);
      else if (hand.x < 0.2 && fabs(hand.z - cube.z) > 0.04) to = cube;
      else to = pv_add(goal, 0.0, 0.0, 0.1);
      if (pv_dxy(hand, obj) > 0.04 || fabs(hand.z - obj.z) > 0.15) grab = -1.0;
      else grab = obj.x < 0.4 ? 0.7 : -1.0;
    } break;
    case T_WINDOW_CLOSE: {                   // sawyer_window_close_v3_policy.py:23-45
      const PV w = pv_add(obj, 0.03, -0.03, -0.08);
      if (pv_dxy(hand, w) > 0.04) to = pv_add(w, 0.0, 0.0, 0.25);
      else if (fabs(hand.z - w.z) > 0.02) to = w;
      else to = pv_add(w, -0.1, 0.0, 0.0);
      grab = 1.0;
    } break;
    case T_WINDOW_OPEN: {                    // sawyer_window_open_v3_policy.py:23-45
      const PV w = pv_add(obj, -0.03, -0.03, -0.08);
      if (pv_dxy(hand, w) > 0.04) to = pv_add(w, 0.0, 0.0, 0.3);
      else if (fabs(hand.z - w.z) > 0.02) to = w;
      else to = pv_add(w, 0.1, 0.0, 0.0);
      grab = 1.0;
    } break;
    default:
      a[0] = a[1] = a[2] = a[3] = NAN;
      return;
  }
  a[0] = (float)(p * (to.x - hand.x));
  a[1] = (float)(p * (to.y - hand.y));
  a[2] = (float)(p * (to.z - hand.z));
  a[3] = (float)grab;
}
