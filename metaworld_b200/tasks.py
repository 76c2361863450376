"""Host-side task registry: everything about a Meta-World V3 task that is not physics.

One `TaskSpec` per reference env class (metaworld/envs/sawyer_*_v3.py): the MJCF file, the static body
its ``reset_model`` moves, the named frames its observation / reward code reads (-> device frame slots
F_TASK0..), the constants from its ``__init__`` (hand_init_pos, hand/goal boxes, random reset space), its
rand_vec rejection rule, and ``task_id`` which selects the device obs / reward / reset code
(csrc/mw_tasks_gen.cuh).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class TaskSpec:
    name: str
    task_id: int
    xml: str
    movable: str | None          # static body whose model.body(name).pos the task's reset_model rewrites
    frames: list                 # [(kind, name)] -> device frame slots F_TASK0 + i
    hand_init_pos: tuple
    hand_low: tuple              # mocap_low/high default to hand_low/high (sawyer_xyz_env.py:196-201)
    hand_high: tuple
    rand_lo: tuple               # _random_reset_space
    rand_hi: tuple
    goal_low: tuple              # goal_space (obs clipping)
    goal_high: tuple
    reject: tuple | None = None  # ((a0,a1),(b0,b1) or fixed point,thr): redraw while |v[a0:a1]-other| < thr
    main_geom: str | None = "objGeom"
    params: tuple = ()
    site_params: tuple = ()      # model.site(name).pos values the task reads (copied into MwTaskConst.p[0:3], [3:6], ...)

    @property
    def rand_low(self):
        return np.asarray(self.rand_lo, dtype=np.float64)

    @property
    def rand_high(self):
        return np.asarray(self.rand_hi, dtype=np.float64)


_OBJ = [("body", "obj"), ("geom", "objGeom")]
_XY = ((0, 2), (3, 5))   # obj xy vs goal xy


def _cat(a, b):
    return tuple(a) + tuple(b)


_BTN = [("body", "button"), ("site", "hole"), ("site", "buttonStart")]
_HL, _HH = (-0.5, 0.40, 0.05), (0.5, 1, 0.5)        # hand_low / hand_high shared by every V3 task
_H0 = (0.0, 0.6, 0.2)

_SPECS = [
    # ---- reach / push / pick-place family (sawyer_reach_v3.py, sawyer_push_v3.py, sawyer_pick_place_v3.py)
    TaskSpec("reach-v3", 0, "sawyer_reach_v3", None, _OBJ, _H0, _HL, _HH,
             _cat((-0.1, 0.6, 0.02), (-0.1, 0.8, 0.05)), _cat((0.1, 0.7, 0.02), (0.1, 0.9, 0.3)),
             (-0.1, 0.8, 0.05), (0.1, 0.9, 0.3), reject=(_XY[0], _XY[1], 0.15)),
    TaskSpec("push-v3", 1, "sawyer_push_v3", None, _OBJ, _H0, _HL, _HH,
             _cat((-0.1, 0.6, 0.02), (-0.1, 0.8, 0.01)), _cat((0.1, 0.7, 0.02), (0.1, 0.9, 0.02)),
             (-0.1, 0.8, 0.01), (0.1, 0.9, 0.02), reject=(_XY[0], _XY[1], 0.15)),
    TaskSpec("pick-place-v3", 2, "sawyer_pick_place_v3", None, _OBJ, _H0, _HL, _HH,
             _cat((-0.1, 0.6, 0.02), (-0.1, 0.8, 0.05)), _cat((0.1, 0.7, 0.02), (0.1, 0.9, 0.3)),
             (-0.1, 0.8, 0.05), (0.1, 0.9, 0.3), reject=(_XY[0], _XY[1], 0.15)),
    # ---- sawyer_door_v3.py (door-open)
    TaskSpec("door-open-v3", 3, "sawyer_door_pull", "door", [("geom", "handle")], _H0, _HL, _HH,
             (0.0, 0.85, 0.15), (0.1, 0.95, 0.15), (-0.3, 0.4, 0.1499), (-0.2, 0.5, 0.1501), main_geom=None),
    # ---- sawyer_drawer_open_v3.py / sawyer_drawer_close_v3.py  (goal_space = hand box)
    TaskSpec("drawer-open-v3", 4, "sawyer_drawer", "drawer", [("body", "drawer_link")], _H0, _HL, _HH,
             (-0.1, 0.9, 0.0), (0.1, 0.9, 0.0), _HL, _HH),
    TaskSpec("drawer-close-v3", 5, "sawyer_drawer", "drawer", [("body", "drawer_link")], _H0, _HL, _HH,
             (-0.1, 0.9, 0.0), (0.1, 0.9, 0.0), _HL, _HH),
    # ---- sawyer_button_press_topdown_v3.py
    TaskSpec("button-press-topdown-v3", 6, "sawyer_button_press_topdown", "box",
             [("body", "button"), ("site", "hole"), ("site", "buttonStart")], (0, 0.4, 0.2), _HL, _HH,
             (-0.1, 0.8, 0.115), (0.1, 0.9, 0.115), _HL, _HH, main_geom="btnGeom"),
    # ---- sawyer_peg_insertion_side_v3.py
    TaskSpec("peg-insert-side-v3", 7, "sawyer_peg_insertion_side", "box",
             [("site", "pegGrasp"), ("site", "pegHead"), ("body", "peg"),
              ("site", "bottom_right_corner_collision_box_1"), ("site", "top_left_corner_collision_box_1"),
              ("site", "bottom_right_corner_collision_box_2"), ("site", "top_left_corner_collision_box_2")],
             _H0, _HL, _HH, _cat((0.0, 0.5, 0.02), (-0.35, 0.4, -0.001)), _cat((0.2, 0.7, 0.02), (-0.25, 0.7, 0.001)),
             (-0.32, 0.4, 0.129), (-0.22, 0.7, 0.131), reject=(_XY[0], _XY[1], 0.1), main_geom=None),
    # ---- sawyer_window_open_v3.py / sawyer_window_close_v3.py
    TaskSpec("window-open-v3", 8, "sawyer_window_horizontal", "window", [("site", "handleOpenStart")], (0, 0.4, 0.2), _HL, _HH,
             (-0.1, 0.7, 0.16), (0.1, 0.9, 0.16), _HL, _HH, main_geom=None),
    TaskSpec("window-close-v3", 9, "sawyer_window_horizontal", "window", [("site", "handleCloseStart")], (0, 0.4, 0.2), _HL, _HH,
             (0.0, 0.75, 0.2), (0.0, 0.9, 0.2), _HL, _HH, main_geom=None),
    # ---- wall variants (sawyer_reach_wall_v3.py, sawyer_push_wall_v3.py, sawyer_pick_place_wall_v3.py)
    TaskSpec("reach-wall-v3", 10, "sawyer_reach_wall_v3", None, _OBJ, _H0, _HL, _HH,
             _cat((-0.05, 0.6, 0.015), (-0.05, 0.85, 0.05)), _cat((0.05, 0.65, 0.015), (0.05, 0.9, 0.3)),
             (-0.05, 0.85, 0.05), (0.05, 0.9, 0.3), reject=(_XY[0], _XY[1], 0.15)),
    TaskSpec("push-wall-v3", 11, "sawyer_push_wall_v3", None, _OBJ, _H0, _HL, _HH,
             _cat((-0.05, 0.6, 0.015), (-0.05, 0.85, 0.01)), _cat((0.05, 0.65, 0.015), (0.05, 0.9, 0.02)),
             (-0.05, 0.85, 0.01), (0.05, 0.9, 0.02), reject=(_XY[0], _XY[1], 0.15)),
    TaskSpec("pick-place-wall-v3", 12, "sawyer_pick_place_wall_v3", None, _OBJ, _H0, _HL, _HH,
             _cat((-0.05, 0.6, 0.015), (-0.05, 0.85, 0.05)), _cat((0.05, 0.65, 0.015), (0.05, 0.9, 0.3)),
             (-0.05, 0.85, 0.05), (0.05, 0.9, 0.3), reject=(_XY[0], _XY[1], 0.15)),
    # ---- sawyer_push_back_v3.py, sawyer_sweep_v3.py, sawyer_sweep_into_goal_v3.py
    TaskSpec("push-back-v3", 13, "sawyer_push_back_v3", None, _OBJ, _H0, _HL, _HH,
             _cat((-0.1, 0.8, 0.02), (-0.1, 0.6, 0.0199)), _cat((0.1, 0.85, 0.02), (0.1, 0.7, 0.0201)),
             (-0.1, 0.6, 0.0199), (0.1, 0.7, 0.0201), reject=(_XY[0], _XY[1], 0.15)),
    TaskSpec("sweep-v3", 14, "sawyer_sweep_v3", None, _OBJ, _H0, _HL, _HH,
             (-0.1, 0.6, 0.02), (0.1, 0.7, 0.02), (0.49, 0.6, 0.00), (0.51, 0.7, 0.02)),
    TaskSpec("sweep-into-v3", 15, "sawyer_table_with_hole", None, _OBJ, _H0, _HL, _HH,
             _cat((-0.1, 0.6, 0.02), (-0.001, 0.8399, 0.0199)), _cat((0.1, 0.7, 0.02), (0.001, 0.8401, 0.0201)),
             (-0.001, 0.8399, 0.0199), (0.001, 0.8401, 0.0201), reject=((0, 2), (0.0, 0.84), 0.15)),
    # ---- sawyer_hand_insert_v3.py, sawyer_pick_out_of_hole_v3.py
    TaskSpec("hand-insert-v3", 16, "sawyer_table_with_hole", None, _OBJ, _H0, (-0.5, 0.40, -0.15), _HH,
             _cat((-0.1, 0.6, 0.05), (-0.04, 0.8, -0.0201)), _cat((0.1, 0.7, 0.05), (0.04, 0.88, -0.0199)),
             (-0.04, 0.8, -0.0201), (0.04, 0.88, -0.0199), reject=(_XY[0], _XY[1], 0.15)),
    TaskSpec("pick-out-of-hole-v3", 17, "sawyer_pick_out_of_hole", None, _OBJ, _H0, (-0.5, 0.40, -0.05), _HH,
             _cat((0, 0.75, 0.02), (-0.1, 0.5, 0.15)), _cat((0, 0.75, 0.02), (0.1, 0.6, 0.3)),
             (-0.1, 0.5, 0.15), (0.1, 0.6, 0.3), reject=(_XY[0], _XY[1], 0.15)),
    # ---- button family (sawyer_button_press_v3.py, ..._wall_v3.py, ..._topdown_wall_v3.py)
    TaskSpec("button-press-v3", 18, "sawyer_button_press", "box", _BTN, (0, 0.4, 0.2), _HL, _HH,
             (-0.1, 0.85, 0.115), (0.1, 0.9, 0.115), _HL, _HH, main_geom="btnGeom"),
    TaskSpec("button-press-wall-v3", 19, "sawyer_button_press_wall", "box", _BTN, (0, 0.4, 0.2), _HL, _HH,
             (-0.05, 0.85, 0.1149), (0.05, 0.9, 0.1151), _HL, _HH, main_geom="btnGeom"),
    TaskSpec("button-press-topdown-wall-v3", 20, "sawyer_button_press_topdown_wall", "box", _BTN, (0, 0.4, 0.2), _HL, _HH,
             (-0.1, 0.8, 0.115), (0.1, 0.9, 0.115), _HL, _HH, main_geom="btnGeom"),
    # ---- coffee family (sawyer_coffee_button_v3.py, sawyer_coffee_pull_v3.py, sawyer_coffee_push_v3.py); mug joint precedes the robot
    TaskSpec("coffee-button-v3", 21, "sawyer_coffee", "coffee_machine", [("site", "buttonStart")], (0.0, 0.4, 0.2), _HL, _HH,
             (-0.1, 0.8, -0.001), (0.1, 0.9, 0.001), (-0.101, 0.61, 0.298), (0.101, 0.71, 0.302), main_geom=None),
    TaskSpec("coffee-pull-v3", 22, "sawyer_coffee", "coffee_machine", [("body", "obj"), ("geom", "mug")], (0.0, 0.4, 0.2), _HL, _HH,
             _cat((-0.05, 0.7, -0.001), (-0.1, 0.55, -0.001)), _cat((0.05, 0.75, 0.001), (0.1, 0.65, 0.001)),
             (-0.1, 0.55, -0.001), (0.1, 0.65, 0.001), reject=(_XY[0], _XY[1], 0.15), main_geom="mug"),
    TaskSpec("coffee-push-v3", 23, "sawyer_coffee", "coffee_machine", [("body", "obj"), ("geom", "mug")], (0.0, 0.4, 0.2), _HL, _HH,
             _cat((-0.1, 0.55, -0.001), (-0.05, 0.7, -0.001)), _cat((0.1, 0.65, 0.001), (0.05, 0.75, 0.001)),
             (-0.05, 0.7, -0.001), (0.05, 0.75, 0.001), reject=(_XY[0], _XY[1], 0.15), main_geom="mug"),
    # ---- sawyer_dial_turn_v3.py
    TaskSpec("dial-turn-v3", 24, "sawyer_dial", "dial", [("body", "dial")], _H0, _HL, _HH,
             (-0.1, 0.7, 0.0), (0.1, 0.8, 0.0), (-0.1, 0.73, 0.0299), (0.1, 0.83, 0.0301), main_geom=None),
    # ---- door family (sawyer_door_close_v3.py, sawyer_door_lock_v3.py, sawyer_door_unlock_v3.py)
    TaskSpec("door-close-v3", 25, "sawyer_door_pull", "door", [("geom", "handle")], (-0.5, 0.6, 0.2), _HL, _HH,
             (0.0, 0.85, 0.15), (0.1, 0.95, 0.15), (0.2, 0.65, 0.1499), (0.3, 0.75, 0.1501), main_geom=None),
    TaskSpec("door-lock-v3", 26, "sawyer_door_lock", "door", [("site", "lockStartLock"), ("body", "door_link"), ("body", "lock_link")],
             _H0, (-0.5, 0.40, -0.15), _HH, (-0.1, 0.8, 0.15), (0.1, 0.85, 0.15), (-0.5, 0.40, -0.15), _HH, main_geom=None),
    TaskSpec("door-unlock-v3", 27, "sawyer_door_lock", "door", [("site", "lockStartUnlock"), ("body", "door_link"), ("body", "lock_link")],
             _H0, (-0.5, 0.40, -0.15), _HH, (-0.1, 0.8, 0.15), (0.1, 0.85, 0.15), (0.0, 0.64, 0.2100), (0.2, 0.7, 0.2111), main_geom=None),
    # ---- sawyer_assembly_peg_v3.py / sawyer_disassemble_peg_v3.py
    TaskSpec("assembly-v3", 28, "sawyer_assembly_peg", "peg", [("site", "RoundNut-8"), ("body", "RoundNut"), ("site", "RoundNut")], _H0, _HL, _HH,
             _cat((0, 0.6, 0.02), (-0.1, 0.75, 0.1)), _cat((0, 0.6, 0.02), (0.1, 0.85, 0.1)),
             (-0.1, 0.75, 0.1), (0.1, 0.85, 0.1), reject=(_XY[0], _XY[1], 0.1), main_geom="WrenchHandle"),
    TaskSpec("disassemble-v3", 29, "sawyer_assembly_peg", "peg", [("site", "RoundNut-8"), ("body", "RoundNut"), ("site", "RoundNut")], (0, 0.4, 0.2), _HL, _HH,
             _cat((0.0, 0.6, 0.025), (-0.1, 0.6, 0.1699)), _cat((0.1, 0.75, 0.02501), (0.1, 0.75, 0.1701)),
             (-0.1, 0.6, 0.1749), (0.1, 0.75, 0.1751), reject=(_XY[0], _XY[1], 0.1), main_geom="WrenchHandle"),
    # ---- sawyer_basketball_v3.py
    TaskSpec("basketball-v3", 30, "sawyer_basketball", "basket_goal", [("body", "bsktball"), ("site", "goal")], _H0, _HL, _HH,
             _cat((-0.1, 0.6, 0.0299), (-0.1, 0.85, 0.0)), _cat((0.1, 0.7, 0.0301), (0.1, 0.9 + 1e-7, 0.0)),
             (-0.1, 0.767, 0.2499), (0.1, 0.817 + 1e-7, 0.2501), reject=(_XY[0], _XY[1], 0.15)),
    # ---- sawyer_bin_picking_v3.py
    TaskSpec("bin-picking-v3", 31, "sawyer_bin_picking", None, [("body", "obj"), ("body", "bin_goal")], _H0, (-0.5, 0.40, 0.07), _HH,
             _cat((-0.21, 0.65, 0.02), (0.1199, 0.699, -0.001)), _cat((-0.03, 0.75, 0.02), (0.1201, 0.701, 0.001)),
             (0.1199, 0.699, -0.001), (0.1201, 0.701, 0.001)),
    # ---- sawyer_box_close_v3.py
    TaskSpec("box-close-v3", 32, "sawyer_box", "boxbody", [("body", "top_link"), ("body", "boxbody")], _H0, _HL, _HH,
             _cat((-0.05, 0.5, 0.02), (-0.1, 0.7, 0.133)), _cat((0.05, 0.55, 0.02), (0.1, 0.8, 0.133)),
             (-0.1, 0.7, 0.133), (0.1, 0.8, 0.133), reject=(_XY[0], _XY[1], 0.25), main_geom="BoxHandleGeom"),
    # ---- sawyer_faucet_open_v3.py / sawyer_faucet_close_v3.py
    TaskSpec("faucet-open-v3", 33, "sawyer_faucet", "faucetBase", [("site", "handleStartOpen"), ("body", "faucetBase")], (0.0, 0.4, 0.2),
             (-0.5, 0.40, -0.15), _HH, (-0.05, 0.8, 0.0), (0.05, 0.85, 0.0), (-0.5, 0.40, -0.15), _HH, main_geom=None),
    TaskSpec("faucet-close-v3", 34, "sawyer_faucet", "faucetBase", [("site", "handleStartClose"), ("body", "faucetBase")], (0.0, 0.4, 0.2),
             (-0.5, 0.40, -0.15), _HH, (-0.1, 0.8, 0.0), (0.1, 0.85, 0.0), (-0.5, 0.40, -0.15), _HH, main_geom=None),
    # ---- sawyer_hammer_v3.py
    TaskSpec("hammer-v3", 35, "sawyer_hammer", "box", [("body", "hammer"), ("body", "nail_link"), ("site", "goal"), ("site", "nailHead")], (0, 0.4, 0.2), _HL, _HH,
             (-0.1, 0.4, 0.0), (0.1, 0.5, 0.0), (0.2399, 0.7399, 0.109), (0.2401, 0.7401, 0.111), main_geom="HammerHandle"),
    # ---- handle family (sawyer_handle_press_v3.py, _press_side, _pull, _pull_side)
    TaskSpec("handle-press-v3", 36, "sawyer_handle_press", "box", [("site", "handleStart"), ("site", "goalPress")], _H0, _HL, _HH,
             (-0.1, 0.8, -0.001), (0.1, 0.9, 0.001), (-0.1, 0.55, 0.04), (0.1, 0.70, 0.08), main_geom=None),
    TaskSpec("handle-press-side-v3", 37, "sawyer_handle_press_sideways", "box", [("site", "handleStart"), ("site", "goalPress")], _H0, _HL, _HH,
             (-0.35, 0.65, -0.001), (-0.25, 0.75, 0.001), _HL, _HH, main_geom=None),
    TaskSpec("handle-pull-v3", 38, "sawyer_handle_press", "box", [("site", "handleRight"), ("site", "goalPull")], _H0, _HL, _HH,
             (-0.1, 0.8, -0.001), (0.1, 0.9, 0.001), (-0.1, 0.55, 0.04), (0.1, 0.70, 0.18), main_geom=None),
    TaskSpec("handle-pull-side-v3", 39, "sawyer_handle_press_sideways", "box", [("site", "handleCenter"), ("site", "goalPull")], _H0, _HL, _HH,
             (-0.35, 0.65, 0.0), (-0.25, 0.75, 0.0), _HL, _HH, main_geom=None),
    # ---- sawyer_lever_pull_v3.py
    TaskSpec("lever-pull-v3", 40, "sawyer_lever_pull", "lever", [("site", "leverStart"), ("geom", "objGeom")], (0, 0.4, 0.2), (-0.5, 0.40, -0.15), _HH,
             (-0.1, 0.7, 0.0), (0.1, 0.8, 0.0), (-0.5, 0.40, -0.15), _HH, main_geom=None),
    # ---- sawyer_peg_unplug_side_v3.py
    TaskSpec("peg-unplug-side-v3", 41, "sawyer_peg_unplug_side", "box", [("site", "pegEnd"), ("body", "plug1")], _H0, _HL, _HH,
             (-0.25, 0.6, -0.001), (-0.15, 0.8, 0.001), (-0.056, 0.6, 0.13), (0.044, 0.8, 0.132), main_geom=None),
    # ---- plate-slide family (sawyer_plate_slide_v3.py, _side, _back, _back_side)
    TaskSpec("plate-slide-v3", 42, "sawyer_plate_slide", "puck_goal", [("geom", "puck")], _H0, _HL, _HH,
             _cat((0.0, 0.6, 0.0), (-0.1, 0.85, 0.0)), _cat((0.0, 0.6, 0.0), (0.1, 0.9, 0.0)), (-0.1, 0.85, 0.0), (0.1, 0.9, 0.0), main_geom=None),
    TaskSpec("plate-slide-side-v3", 43, "sawyer_plate_slide_sideway", "puck_goal", [("geom", "puck")], _H0, _HL, _HH,
             _cat((0.0, 0.6, 0.0), (-0.3, 0.54, 0.0)), _cat((0.0, 0.6, 0.0), (-0.25, 0.66, 0.0)), (-0.3, 0.54, 0.0), (-0.25, 0.66, 0.0), main_geom=None),
    TaskSpec("plate-slide-back-v3", 44, "sawyer_plate_slide", "puck_goal", [("geom", "puck")], _H0, _HL, _HH,
             _cat((0.0, 0.85, 0.0), (-0.1, 0.6, 0.015)), _cat((0.0, 0.85, 0.0), (0.1, 0.6, 0.015)), (-0.1, 0.6, 0.015), (0.1, 0.6, 0.015), main_geom=None),
    TaskSpec("plate-slide-back-side-v3", 45, "sawyer_plate_slide_sideway", "puck_goal", [("geom", "puck")], _H0, _HL, _HH,
             _cat((-0.25, 0.6, 0.0), (-0.05, 0.6, 0.015)), _cat((-0.25, 0.6, 0.0), (0.15, 0.6, 0.015)), (-0.05, 0.6, 0.015), (0.15, 0.6, 0.015), main_geom=None),
    # ---- sawyer_shelf_place_v3.py
    TaskSpec("shelf-place-v3", 46, "sawyer_shelf_placing", "shelf", _OBJ, _H0, _HL, _HH,
             _cat((-0.1, 0.5, 0.019), (-0.1, 0.8, 0.299)), _cat((0.1, 0.6, 0.021), (0.1, 0.9, 0.301)),
             (-0.1, 0.8, 0.299), (0.1, 0.9, 0.301), reject=(_XY[0], _XY[1], 0.1), site_params=("goal",)),
    # ---- sawyer_soccer_v3.py
    TaskSpec("soccer-v3", 47, "sawyer_soccer", "goal_whole", [("body", "soccer_ball")], _H0, _HL, _HH,
             _cat((-0.1, 0.6, 0.03), (-0.1, 0.8, 0.0)), _cat((0.1, 0.7, 0.03), (0.1, 0.9, 0.0)), (-0.1, 0.8, 0.0), (0.1, 0.9, 0.0),
             reject=(_XY[0], _XY[1], 0.15)),
    # ---- sawyer_stick_push_v3.py / sawyer_stick_pull_v3.py
    TaskSpec("stick-push-v3", 48, "sawyer_stick_obj", None, [("body", "stick"), ("site", "insertion"), ("body", "object"), ("site", "stick_end")],
             _H0, _HL, _HH, _cat((-0.08, 0.58, 0.0), (0.399, 0.55, 0.1319)), _cat((-0.03, 0.62, 0.001), (0.401, 0.6, 0.1321)),
             (0.399, 0.55, 0.1319), (0.401, 0.6, 0.1321), reject=(_XY[0], _XY[1], 0.1)),
    TaskSpec("stick-pull-v3", 49, "sawyer_stick_obj", None, [("body", "stick"), ("site", "insertion"), ("body", "object"), ("site", "stick_end")],
             _H0, (-0.5, 0.35, 0.05), _HH, _cat((-0.1, 0.55, 0.0), (0.35, 0.45, 0.0199)), _cat((0.0, 0.65, 0.001), (0.45, 0.55, 0.0201)),
             (0.35, 0.45, 0.0199), (0.45, 0.55, 0.0201), reject=(_XY[0], _XY[1], 0.1)),
]

TASKS = {t.name: t for t in _SPECS}
TASK_IDS = {t.name: t.task_id for t in _SPECS}

# What each reference class's `_get_id_main_object()` does (SawyerXYZEnv default: data.geom("objGeom").id,
# sawyer_xyz_env.py:442-443, and the per-task overrides): None = returns None; otherwise (geom name, lookup), where
# lookup "name2id" is `model.geom_name2id(...)`, which MuJoCo's Python bindings do not have (the reference raises
# AttributeError), and "geom" is `data.geom(name).id` / `model.geom(name).id` (KeyError when the model has no such geom).
_NAME2ID = ("drawer-open-v3", "button-press-topdown-v3", "pick-out-of-hole-v3", "button-press-v3", "button-press-wall-v3",
            "button-press-topdown-wall-v3", "assembly-v3", "disassemble-v3", "basketball-v3", "bin-picking-v3",
            "box-close-v3", "hammer-v3", "lever-pull-v3")
_MAIN_GEOM = {"button-press-topdown-v3": "btnGeom", "button-press-v3": "btnGeom", "button-press-wall-v3": "btnGeom",
              "button-press-topdown-wall-v3": "btnGeom", "coffee-pull-v3": "mug", "coffee-push-v3": "mug",
              "assembly-v3": "WrenchHandle", "disassemble-v3": "WrenchHandle", "box-close-v3": "BoxHandleGeom",
              "hammer-v3": "HammerHandle"}
# frames whose position a task keeps equal to its _target_pos after every forward pass (csrc/mw_tasks_gen.cuh
# task_live_update): basketball's _target_pos aliases data.site("goal").xpos
TARGET_ALIAS = {"basketball-v3": (("site", "goal"),)}
# sites whose model.site(name).pos a task's reset_model sets to a per-episode vector (e.g. sawyer_reach_v3.py:134): the
# site then sits at (its body's position) + that vector.  "target": _target_pos; ("obj_init", offset): obj_init_pos +
# offset (sawyer_disassemble_peg_v3.py:128-131).  Basketball's goal is live instead (TARGET_ALIAS); shelf-place writes the
# site's xpos only (_set_pos_site), which the next forward pass undoes.
_GOAL_IS_TARGET = ("reach-v3", "push-v3", "pick-place-v3", "door-open-v3", "drawer-open-v3", "drawer-close-v3",
                   "peg-insert-side-v3", "window-open-v3", "window-close-v3", "reach-wall-v3", "push-wall-v3",
                   "pick-place-wall-v3", "push-back-v3", "sweep-v3", "sweep-into-v3", "hand-insert-v3", "pick-out-of-hole-v3",
                   "dial-turn-v3", "door-close-v3", "box-close-v3", "lever-pull-v3", "peg-unplug-side-v3", "plate-slide-v3",
                   "plate-slide-side-v3", "plate-slide-back-v3", "plate-slide-back-side-v3", "soccer-v3", "stick-push-v3",
                   "stick-pull-v3")
MOVED_SITES = {**{t: {"goal": "target"} for t in _GOAL_IS_TARGET},
               "coffee-pull-v3": {"mug_goal": "target"}, "coffee-push-v3": {"mug_goal": "target"},
               "faucet-open-v3": {"goal_open": ("obj_init", (0.175, 0.0, 0.125))},      # sawyer_faucet_open_v3.py:111-114
               "faucet-close-v3": {"goal_close": ("obj_init", (-0.175, 0.0, 0.125))},   # sawyer_faucet_close_v3.py
               "assembly-v3": {"pegTop": "target"}, "disassemble-v3": {"pegTop": ("obj_init", (0.0, 0.0, 0.08))}}
# tasks whose _get_obs_dict() overrides state_achieved_goal (default: obs[3:-3]): a (kind, name, offset) frame position,
# or "objects" = _get_pos_objects() (sawyer_assembly_peg_v3.py:110-113, sawyer_disassemble_peg_v3.py:111-114,
# sawyer_stick_push_v3.py:126-131, sawyer_stick_pull_v3.py:131-134, sawyer_plate_slide_back_side_v3.py:114-119)
ACHIEVED_GOAL = {"assembly-v3": ("body", "RoundNut", None), "disassemble-v3": ("body", "RoundNut", None),
                 "stick-push-v3": ("site", "insertion", (0.0, 0.09, 0.0)), "stick-pull-v3": ("site", "insertion", None),
                 "plate-slide-back-side-v3": "objects"}
MAIN_OBJECT = {t.name: None if t.name in ("door-lock-v3", "door-unlock-v3", "coffee-button-v3")
               else (_MAIN_GEOM.get(t.name, "objGeom"), "name2id" if t.name in _NAME2ID else "geom") for t in _SPECS}
assert sorted(TASK_IDS.values()) == list(range(len(_SPECS)))


def enum_name(name: str) -> str:
    return "T_" + name[:-3].upper().replace("-", "_")


def emit_task_enum() -> str:
    """C enum of task ids for csrc/mw_tasks_gen.cuh (written by build.write_header)."""
    lines = ["/* GENERATED by metaworld_b200/tasks.py:emit_task_enum -- do not edit. */", "#pragma once", "enum {"]
    for t in sorted(_SPECS, key=lambda t: t.task_id):
        lines.append(f"  {enum_name(t.name)} = {t.task_id},")
    lines += ["  T_NTASK", "};"]
    return "\n".join(lines) + "\n"
