"""Lowering: mjModel-like tables (`mjcf.Model`) -> flat device blob (`MwModel`).

What the reference keeps in ``mjModel`` (36-38 bodies, 37-69 geoms) is reduced
to what the step kernel touches:

* **links**  : one per jointed body; jointless descendants (hand, pads, sensors)
  are folded into their link (inertia merged, geoms / frames re-expressed in the
  link frame).  Sawyer = 9 links; tasks add 1-2.
* **static geometry** is folded into the world.  Each model has at most one
  static body whose ``model.body(name).pos`` the task's ``reset_model`` rewrites
  (e.g. ``drawer``, ``door``, ``box``; reference: metaworld/envs/*.py) -- its
  subtree is tagged ``shift`` and the per-env translation is applied at run time.
* **colliders**: only geoms that appear in at least one candidate pair after
  MuJoCo's static filters (same/parent weld body, contype/conaffinity).
* **pairs** carry an index into a small table of pre-mixed contact parameters
  (condim/friction/solref/solimp/margin mixing is a pure function of the two
  geoms).
* **frames**: the named bodies / geoms / sites that observations and rewards read.

The struct layout below is the single source of truth: `emit_header()` writes
``csrc/mw_model.h`` from it and `pack()` fills a numpy record with the same
layout, which is copied verbatim to the GPU and staged into shared memory.
"""
from __future__ import annotations

import numpy as np

from . import mjcf
from .mjcf import (GEOM_BOX, GEOM_CAPSULE, GEOM_MESH, GEOM_PLANE, GEOM_SPHERE, JNT_FREE, JNT_HINGE, JNT_SLIDE, quat2mat,
                   quat_conj, quat_mul, quat_norm)

MAXLINK, MAXDOF, MAXNQ, MAXGEOM, MAXPAIR, MAXPARAM, MAXFRAME = 12, 17, 18, 40, 384, 32, 32
NPARAM = 12
MAXCONV = 128        # general convex pairs per model (the separating-axis hint table's row length; MT50 maximum: hammer)
NO_CSLOT = 255       # pair_cslot of a pair that never goes to GJK/EPA

# (name, ctype, shape)
FIELDS = [
    ("qpos0d", "f8", (MAXNQ,)),     # float64 copy of qpos0 (mj_resetData must reproduce free-joint initial poses exactly)
    ("nlink", "i4", ()), ("nq", "i4", ()), ("nv", "i4", ()), ("ngeom", "i4", ()), ("npair", "i4", ()),
    ("nframe", "i4", ()), ("nmeshvert", "i4", ()),
    ("ndepth", "i4", ()),           # levels of the link forest: 1 + the largest link_depth
    ("timestep", "f4", ()), ("solver_scale", "f4", ()), ("gravity", "f4", (3,)), ("tolerance", "f4", ()),
    ("impratio", "f4", ()), ("pad1", "f4", ()),
    # links
    ("link_parent", "i4", (MAXLINK,)), ("link_jtype", "i4", (MAXLINK,)), ("link_qadr", "i4", (MAXLINK,)),
    ("link_dadr", "i4", (MAXLINK,)), ("link_shift", "i4", (MAXLINK,)), ("link_dofmask", "u4", (MAXLINK,)),
    ("link_depth", "i4", (MAXLINK,)),       # 0 for a root link, parent's + 1 otherwise (parents precede their children)
    ("link_pos", "f4", (MAXLINK, 3)), ("link_quat", "f4", (MAXLINK, 4)), ("link_jaxis", "f4", (MAXLINK, 3)),
    ("link_jpos", "f4", (MAXLINK, 3)), ("link_mass", "f4", (MAXLINK,)), ("link_com", "f4", (MAXLINK, 3)),
    ("link_inertia", "f4", (MAXLINK, 6)),
    # dofs
    ("dof_link", "i4", (MAXDOF,)), ("dof_qadr", "i4", (MAXDOF,)), ("dof_limited", "i4", (MAXDOF,)),
    ("dof_damping", "f4", (MAXDOF,)), ("dof_armature", "f4", (MAXDOF,)), ("dof_invweight", "f4", (MAXDOF,)),
    ("dof_lo", "f4", (MAXDOF,)), ("dof_hi", "f4", (MAXDOF,)), ("dof_stiffness", "f4", (MAXDOF,)),
    ("dof_springref", "f4", (MAXDOF,)), ("qpos0", "f4", (MAXNQ,)),
    # two position actuators (fingers): dof, kp, ctrl range
    ("act_dof", "i4", (2,)), ("act_kp", "f4", (2,)), ("act_lo", "f4", (2,)), ("act_hi", "f4", (2,)),
    # mocap weld (body2 = hand)
    ("weld_link", "i4", ()), ("weld_pos", "f4", (3,)), ("weld_quat", "f4", (4,)), ("weld_invw", "f4", (2,)),
    ("weld_solref", "f4", (2,)), ("weld_solimp", "f4", (5,)), ("weld_torquescale", "f4", ()),
    ("mocap_pos0", "f4", (3,)), ("mocap_quat0", "f4", (4,)),
    # colliders
    ("geom_type", "i4", (MAXGEOM,)), ("geom_link", "i4", (MAXGEOM,)), ("geom_shift", "i4", (MAXGEOM,)),
    ("geom_meshadr", "i4", (MAXGEOM,)), ("geom_meshnum", "i4", (MAXGEOM,)), ("geom_srcid", "i4", (MAXGEOM,)),
    ("geom_pos", "f4", (MAXGEOM, 3)), ("geom_mat", "f4", (MAXGEOM, 9)), ("geom_size", "f4", (MAXGEOM, 3)),
    ("geom_rbound", "f4", (MAXGEOM,)), ("geom_invw", "f4", (MAXGEOM, 2)),
    ("geom_aabb", "f4", (MAXGEOM, 6)),      # bounding box in the geom frame: centre xyz, half extents xyz (broadphase only)
    # candidate pairs + pre-mixed contact parameters
    ("pair_g1", "u1", (MAXPAIR,)), ("pair_g2", "u1", (MAXPAIR,)), ("pair_param", "u1", (MAXPAIR,)),
    ("pair_cslot", "u1", (MAXPAIR,)),       # slot among the model's general convex pairs (GJK/EPA candidates), else NO_CSLOT
    ("param", "f4", (MAXPARAM, NPARAM)),
    # frames read by obs / reward code
    ("frame_link", "i4", (MAXFRAME,)), ("frame_shift", "i4", (MAXFRAME,)), ("frame_pos", "f4", (MAXFRAME, 3)),
    ("frame_quat", "f4", (MAXFRAME, 4)),
]
# param row: margin, includemargin, dim, fr_slide, fr_spin, solref0, solref1, solimp0, solimp1, solimp2, solimp3, solimp4

DTYPE = np.dtype([(n, t, s) for n, t, s in FIELDS], align=True)

# one record of an mw_query frame table (MwQueryFrame in csrc/mw_engine.cu)
QUERY_DTYPE = np.dtype([("link", "i4"), ("flags", "i4"), ("pos", "f8", 3), ("quat", "f8", 4)])
QF_SHIFT, QF_MISSING, QF_TARGET, QF_ADD_TARGET, QF_ADD_OBJ_INIT = 1, 2, 4, 8, 16
MOCAP_LINK = -2      # query-table link of a frame on the mocap body (posed by the env's mocap target)

# robot frames every task uses (indices are fixed; task frames follow)
ROBOT_FRAMES = [("body", "hand"), ("body", "rightclaw"), ("body", "leftclaw"), ("body", "rightpad"),
                ("body", "leftpad"), ("site", "rightEndEffector"), ("site", "leftEndEffector")]
F_HAND, F_RCLAW, F_LCLAW, F_RPAD, F_LPAD, F_REE, F_LEE, F_TASK0 = range(8)


def emit_header() -> str:
    ctype = {"i4": "int", "u4": "unsigned int", "f4": "float", "u1": "unsigned char", "f8": "double"}
    lines = ["/* GENERATED by metaworld_b200/lower.py:emit_header -- do not edit. */", "#pragma once",
             f"#define MW_MAXLINK {MAXLINK}", f"#define MW_MAXDOF {MAXDOF}", f"#define MW_MAXNQ {MAXNQ}",
             f"#define MW_MAXGEOM {MAXGEOM}", f"#define MW_MAXPAIR {MAXPAIR}", f"#define MW_MAXPARAM {MAXPARAM}",
             f"#define MW_MAXFRAME {MAXFRAME}", f"#define MW_NPARAM {NPARAM}", f"#define MW_NCONV {MAXCONV}",
             "struct MwModel {"]
    for n, t, s in FIELDS:
        dims = "".join(f"[{d}]" for d in s)
        lines.append(f"  {ctype[t]} {n}{dims};")
    lines.append("};")
    lines.append(f"static_assert(sizeof(MwModel) == {DTYPE.itemsize}, \"MwModel layout mismatch with lower.py\");")
    for i, nm in enumerate(["F_HAND", "F_RCLAW", "F_LCLAW", "F_RPAD", "F_LPAD", "F_REE", "F_LEE", "F_TASK0"]):
        lines.append(f"#define {nm} {i}")
    return "\n".join(lines) + "\n"


class Lowered:
    def __init__(self):
        self.rec = np.zeros((), dtype=DTYPE)
        self.meshvert = np.zeros((0, 3), dtype=np.float32)
        self.frame_names = []
        self.geom_names = []     # collider index -> source geom name
        self.geom_src = []       # collider index -> source geom id
        self.link_body = []      # link index -> source body id
        self.movable = None
        self._frame_ctx = None   # (model, body pose relative to its link, link of every body, shift flag of every body)

    def resolve_frame(self, kind, name):
        """A ("body" | "site" | "geom", name) frame of the model -> (link, shift flag, pos, quat) relative to the link that
        carries it (link -1: the world, translated at run time by the env's shift when the flag is set; MOCAP_LINK: the
        mocap body, posed by the env's mocap target).  KeyError when the model has no such name."""
        m, rel_pos, rel_quat, link_of_body, shifted = self._frame_ctx
        a = m.arrays
        if kind not in ("body", "site", "geom"):
            raise ValueError(kind)
        if name not in m.names[kind]:
            raise KeyError(f"no {kind} named {name!r}")
        i = m.names[kind].index(name)
        if kind == "body":
            b = i
            fp, fq = rel_pos[b], rel_quat[b]
        else:
            b = a[f"{kind}_bodyid"][i]
            fp, fq = _compose(rel_pos[b], rel_quat[b], a[f"{kind}_pos"][i], a[f"{kind}_quat"][i])
        l = int(link_of_body[b])
        if a["body_mocapid"][b] >= 0:      # a mocap body sits at data.mocap_pos / mocap_quat: the pose is relative to it
            if kind == "body":
                fp, fq = np.zeros(3), np.array([1.0, 0, 0, 0])
            else:
                fp, fq = a[f"{kind}_pos"][i], a[f"{kind}_quat"][i]
            l = MOCAP_LINK
        return l, int(l < 0 and shifted[b]), np.asarray(fp, dtype=np.float64), np.asarray(fq, dtype=np.float64)

    def query_table(self, frames, target_alias=(), moved_sites=None):
        """The mw_query frame records (QUERY_DTYPE) of a list of (kind, name) pairs; a name the model lacks gives a NaN row
        (QF_MISSING).  `target_alias`: the frames whose position the task keeps equal to its _target_pos (QF_TARGET).
        `moved_sites`: {site name: "target" | ("obj_init", offset)} of the sites whose model.site(name).pos the task's
        reset_model sets to a per-episode vector; their row holds the parent body's position (+ offset) and the kernel adds
        the env's vector (QF_ADD_TARGET / QF_ADD_OBJ_INIT)."""
        m, rel_pos, rel_quat, link_of_body, _ = self._frame_ctx
        t = np.zeros(len(frames), dtype=QUERY_DTYPE)
        for k, (kind, name) in enumerate(frames):
            try:
                l, sh, fp, fq = self.resolve_frame(kind, name)
            except KeyError:
                t[k]["link"], t[k]["flags"] = -1, QF_MISSING
                continue
            flags = (QF_SHIFT if sh else 0) | (QF_TARGET if (kind, name) in target_alias else 0)
            move = (moved_sites or {}).get(name) if kind == "site" else None
            if move is not None:
                b = m.arrays["site_bodyid"][m.names["site"].index(name)]
                assert l == -1 and np.allclose(rel_quat[b], [1, 0, 0, 0]), "moved sites sit on static, unrotated bodies"
                fp = rel_pos[b] + (0.0 if move == "target" else np.asarray(move[1], dtype=np.float64))
                flags |= QF_ADD_TARGET if move == "target" else QF_ADD_OBJ_INIT
            t[k]["link"], t[k]["pos"], t[k]["quat"], t[k]["flags"] = l, fp, fq, flags
        return t

    def collider(self, geom_name):
        """Collider index of a source geom (the index touching_object compares contacts against), -1 when the geom takes
        part in no contact pair or does not exist."""
        return self.geom_names.index(geom_name) if geom_name in self.geom_names else -1


def _compose(p1, q1, p2, q2):
    """(p1,q1) o (p2,q2): child pose expressed in the frame p1,q1 is given in."""
    return p1 + quat2mat(q1) @ p2, quat_norm(quat_mul(q1, q2))


def lower(m: mjcf.Model, movable: str | None, task_frames=()) -> Lowered:
    a = m.arrays
    nb = m.nbody
    out = Lowered()
    r = out.rec
    out.movable = movable
    mov_id = m.names["body"].index(movable) if movable else -1
    if mov_id >= 0:
        assert a["body_parentid"][mov_id] == 0 and a["body_weldid"][mov_id] == 0, "movable body must be a static world child"

    # which static bodies ride on the movable body
    shifted = np.zeros(nb, dtype=bool)
    for b in range(1, nb):
        p = a["body_parentid"][b]
        shifted[b] = (b == mov_id) or shifted[p]

    # ---- links: one per joint (free joint = one link with 6 dofs; n slide/hinge joints on a body = n links in series)
    link_of_body = -np.ones(nb, dtype=np.int64)   # link that carries the body's frame (last joint of the weld root)
    links = []                                    # dicts
    # pose of every body relative to its carrying link (or world): computed by walking down
    rel_pos = np.zeros((nb, 3))
    rel_quat = np.tile(np.array([1.0, 0, 0, 0]), (nb, 1))
    for b in range(1, nb):
        p = a["body_parentid"][b]
        # body frame at qpos0 relative to parent's carrying link
        bp, bq = _compose(rel_pos[p], rel_quat[p], a["body_pos"][b], a["body_quat"][b])
        parent_link = link_of_body[p]
        nj = a["body_jntnum"][b]
        if nj == 0:
            link_of_body[b] = parent_link
            rel_pos[b], rel_quat[b] = bp, bq
            continue
        for k in range(nj):
            j = a["body_jntadr"][b] + k
            jt = int(a["jnt_type"][j])
            L = dict(parent=int(parent_link), jtype=jt, qadr=int(a["jnt_qposadr"][j]), dadr=int(a["jnt_dofadr"][j]),
                     shift=int(shifted[p] and parent_link < 0), body=b,
                     pos=bp if k == 0 else np.zeros(3), quat=bq if k == 0 else np.array([1.0, 0, 0, 0]),
                     jaxis=a["jnt_axis"][j].copy(), jpos=a["jnt_pos"][j].copy())
            if jt == JNT_FREE:
                assert parent_link < 0 and nj == 1
            else:
                assert abs(a["qpos0"][L["qadr"]]) == 0.0, "non-zero joint ref not supported"
            links.append(L)
            parent_link = len(links) - 1
        link_of_body[b] = parent_link
        rel_pos[b], rel_quat[b] = np.zeros(3), np.array([1.0, 0, 0, 0])
    nl = len(links)
    assert nl <= MAXLINK, nl
    nv = m.nv
    assert nv <= MAXDOF and m.nq <= MAXNQ

    # ---- inertia folding (into the carrying link frame)
    acc = [dict(m=0.0, mc=np.zeros(3), parts=[]) for _ in range(nl)]
    for b in range(1, nb):
        l = link_of_body[b]
        if l < 0:
            continue
        mass = a["body_mass"][b]
        I = a["body_inertia"][b]
        if mass <= 0 and not np.any(I > 0):
            continue
        cp, cq = _compose(rel_pos[b], rel_quat[b], a["body_ipos"][b], a["body_iquat"][b])
        R = quat2mat(cq)
        acc[l]["m"] += mass
        acc[l]["mc"] += mass * cp
        acc[l]["parts"].append((mass, cp, R @ np.diag(I) @ R.T))
    for l in range(nl):
        L = links[l]
        mtot = acc[l]["m"]
        com = acc[l]["mc"] / mtot if mtot > 0 else np.zeros(3)
        It = np.zeros((3, 3))
        for mass, cp, Iw in acc[l]["parts"]:
            d = cp - com
            It += Iw + mass * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
        r["link_parent"][l] = L["parent"]
        assert L["parent"] < l
        r["link_depth"][l] = 0 if L["parent"] < 0 else r["link_depth"][L["parent"]] + 1
        r["link_jtype"][l] = L["jtype"]
        r["link_qadr"][l] = L["qadr"]
        r["link_dadr"][l] = L["dadr"]
        r["link_shift"][l] = L["shift"]
        r["link_pos"][l] = L["pos"]
        r["link_quat"][l] = L["quat"]
        r["link_jaxis"][l] = L["jaxis"]
        r["link_jpos"][l] = L["jpos"]
        r["link_mass"][l] = mtot
        r["link_com"][l] = com
        r["link_inertia"][l] = [It[0, 0], It[1, 1], It[2, 2], It[0, 1], It[0, 2], It[1, 2]]
        out.link_body.append(L["body"])
    # dof tables
    for l in range(nl):
        L = links[l]
        nd = 6 if L["jtype"] == JNT_FREE else 1
        mask = 0
        c = l
        while c >= 0:
            ndc = 6 if links[c]["jtype"] == JNT_FREE else 1
            for k in range(ndc):
                mask |= 1 << (links[c]["dadr"] + k)
            c = links[c]["parent"]
        r["link_dofmask"][l] = mask
        for k in range(nd):
            d = L["dadr"] + k
            r["dof_link"][d] = l
            r["dof_qadr"][d] = L["qadr"] + k if L["jtype"] != JNT_FREE else L["qadr"] + k  # free: rot dofs map to quat (unused)
    for d in range(nv):
        j = a["dof_jntid"][d]
        r["dof_damping"][d] = a["dof_damping"][d]
        r["dof_armature"][d] = a["dof_armature"][d]
        r["dof_invweight"][d] = a["dof_invweight0"][d]
        lim = bool(a["jnt_limited"][j]) and a["jnt_type"][j] != JNT_FREE
        r["dof_limited"][d] = int(lim)
        r["dof_lo"][d], r["dof_hi"][d] = a["jnt_range"][j]
        r["dof_stiffness"][d] = a["jnt_stiffness"][j] if a["jnt_type"][j] != JNT_FREE else 0.0
        r["dof_springref"][d] = a["qpos_spring"][a["jnt_qposadr"][j]] if a["jnt_type"][j] != JNT_FREE else 0.0
        assert a["jnt_margin"][j] == 0
    r["qpos0"][: m.nq] = a["qpos0"]
    r["qpos0d"][: m.nq] = a["qpos0"]
    r["nlink"], r["nq"], r["nv"] = nl, m.nq, nv
    r["ndepth"] = int(r["link_depth"][:nl].max()) + 1
    r["timestep"] = m.opt["timestep"]
    r["solver_scale"] = 1.0 / (m.opt["meaninertia"] * max(1, nv))
    r["gravity"] = m.opt["gravity"]
    r["tolerance"] = m.opt["tolerance"]
    r["impratio"] = m.opt["impratio"]
    assert m.opt.get("cone") == "elliptic"

    # ---- actuators
    assert len(a["actuator_jntid"]) == 2
    for u in range(2):
        j = a["actuator_jntid"][u]
        r["act_dof"][u] = a["jnt_dofadr"][j]
        r["act_kp"][u] = a["actuator_kp"][u]
        r["act_lo"][u], r["act_hi"][u] = a["actuator_ctrlrange"][u]

    # ---- weld (mocap -> hand).  eq_data after reset_mocap_welds (sawyer_xyz_env.py:133-140)
    assert len(a["eq_obj1id"]) == 1
    b1, b2 = int(a["eq_obj1id"][0]), int(a["eq_obj2id"][0])
    assert a["body_mocapid"][b1] >= 0
    r["weld_link"] = link_of_body[b2]
    r["weld_pos"] = rel_pos[b2]
    r["weld_quat"] = rel_quat[b2]
    r["weld_invw"] = a["body_invweight0"][b1] + a["body_invweight0"][b2]
    r["weld_solref"] = a["eq_solref"][0]
    r["weld_solimp"] = a["eq_solimp"][0]
    r["weld_torquescale"] = 5.0
    r["mocap_pos0"] = a["body_pos"][b1]
    r["mocap_quat0"] = a["body_quat"][b1]

    # ---- candidate pairs (same filters as MuJoCo's mj_collision [3P]) and colliders
    ng = m.ngeom
    pairs = []
    for g1 in range(ng):
        for g2 in range(g1 + 1, ng):
            bb1, bb2 = a["geom_bodyid"][g1], a["geom_bodyid"][g2]
            w1, w2 = a["body_weldid"][bb1], a["body_weldid"][bb2]
            if w1 == w2:
                continue
            p1 = a["body_weldid"][a["body_parentid"][w1]]
            p2 = a["body_weldid"][a["body_parentid"][w2]]
            if w1 != 0 and w2 != 0 and (w1 == p2 or w2 == p1):
                continue
            if not ((a["geom_contype"][g1] & a["geom_conaffinity"][g2]) or (a["geom_contype"][g2] & a["geom_conaffinity"][g1])):
                continue
            if a["geom_type"][g1] <= a["geom_type"][g2]:
                pairs.append((g1, g2))
            else:
                pairs.append((g2, g1))
    used = sorted({g for p in pairs for g in p})
    assert len(used) <= MAXGEOM and len(pairs) <= MAXPAIR, (len(used), len(pairs))
    cid = {g: i for i, g in enumerate(used)}
    mesh_adr = {}
    mv = []
    for i, g in enumerate(used):
        b = a["geom_bodyid"][g]
        l = link_of_body[b]
        gp, gq = _compose(rel_pos[b], rel_quat[b], a["geom_pos"][g], a["geom_quat"][g])
        r["geom_type"][i] = a["geom_type"][g]
        r["geom_link"][i] = l
        r["geom_shift"][i] = int(l < 0 and shifted[b])
        r["geom_pos"][i] = gp
        r["geom_mat"][i] = quat2mat(gq).reshape(-1)
        r["geom_size"][i] = a["geom_size"][g]
        r["geom_rbound"][i] = a["geom_rbound"][g]
        gt, gs = int(a["geom_type"][g]), a["geom_size"][g]
        if gt == GEOM_MESH:
            hv = np.asarray(m.meshes[int(a["geom_dataid"][g])]["vert"], dtype=np.float64)
            lo, hi = hv.min(axis=0), hv.max(axis=0)
            r["geom_aabb"][i] = np.concatenate([(lo + hi) / 2, (hi - lo) / 2 * (1 + 1e-6) + 1e-7])
        elif gt == 6:    # box
            r["geom_aabb"][i] = [0, 0, 0, gs[0], gs[1], gs[2]]
        elif gt == 5:    # cylinder
            r["geom_aabb"][i] = [0, 0, 0, gs[0], gs[0], gs[1]]
        elif gt == 3:    # capsule
            r["geom_aabb"][i] = [0, 0, 0, gs[0], gs[0], gs[1] + gs[0]]
        elif gt == 2:    # sphere
            r["geom_aabb"][i] = [0, 0, 0, gs[0], gs[0], gs[0]]
        else:            # plane and anything else: no box cull
            r["geom_aabb"][i] = [0, 0, 0, 1e9, 1e9, 1e9]
        r["geom_invw"][i] = a["body_invweight0"][b]
        r["geom_srcid"][i] = g
        r["geom_meshadr"][i] = 0
        r["geom_meshnum"][i] = 0
        if a["geom_type"][g] == GEOM_MESH:
            mid = int(a["geom_dataid"][g])
            if mid not in mesh_adr:
                mesh_adr[mid] = sum(len(x) for x in mv)
                mv.append(np.asarray(m.meshes[mid]["vert"], dtype=np.float32))
            r["geom_meshadr"][i] = mesh_adr[mid]
            r["geom_meshnum"][i] = len(m.meshes[mid]["vert"])
        out.geom_names.append(m.names["geom"][g])
        out.geom_src.append(g)
    r["ngeom"] = len(used)
    out.meshvert = np.concatenate(mv, axis=0) if mv else np.zeros((0, 3), dtype=np.float32)
    r["nmeshvert"] = len(out.meshvert)

    params = []
    nconv = 0
    for k, (g1, g2) in enumerate(pairs):
        prm = mix_params(a, g1, g2)
        key = tuple(np.round(prm, 12))
        if key not in params:
            params.append(key)
        r["pair_g1"][k], r["pair_g2"][k], r["pair_param"][k] = cid[g1], cid[g2], params.index(key)
        r["pair_cslot"][k] = NO_CSLOT
        if general_convex(a["geom_type"][g1], a["geom_type"][g2]):
            r["pair_cslot"][k] = nconv
            nconv += 1
    assert len(params) <= MAXPARAM, len(params)
    assert nconv <= MAXCONV, nconv
    for i, p in enumerate(params):
        r["param"][i] = p
    r["npair"] = len(pairs)

    # ---- frames
    out._frame_ctx = (m, rel_pos, rel_quat, link_of_body, shifted)
    frames = list(ROBOT_FRAMES) + list(task_frames)
    assert len(frames) <= MAXFRAME
    for i, (kind, name) in enumerate(frames):
        l, sh, fp, fq = out.resolve_frame(kind, name)
        assert l != MOCAP_LINK, "the step kernels read no frame on the mocap body"
        r["frame_link"][i] = l
        r["frame_shift"][i] = sh
        r["frame_pos"][i] = fp
        r["frame_quat"][i] = fq
        out.frame_names.append((kind, name))
    r["nframe"] = len(frames)
    return out


def general_convex(t1, t2) -> bool:
    """Whether the narrowphase may send a pair (t1 <= t2) to GJK/EPA: everything but the analytic pairs (plane-*, and any
    two of sphere / capsule / box; csrc/mw_collide.cuh pair_is_analytic) and plane-mesh, which is one support query.
    Cylinder-box and cylinder-cylinder pairs count: they go to GJK/EPA whenever their axes are not aligned."""
    analytic3 = (GEOM_SPHERE, GEOM_CAPSULE, GEOM_BOX)
    return t1 != GEOM_PLANE and not (t1 in analytic3 and t2 in analytic3)


def mix_params(a, g1, g2):
    """Contact parameter mixing for a geom pair (MuJoCo mj_contactParam [3P]; priorities are all 0 here)."""
    assert a["geom_priority"][g1] == a["geom_priority"][g2]
    margin = max(a["geom_margin"][g1], a["geom_margin"][g2])
    gap = max(a["geom_gap"][g1], a["geom_gap"][g2])
    dim = max(a["geom_condim"][g1], a["geom_condim"][g2])
    s1, s2 = a["geom_solmix"][g1], a["geom_solmix"][g2]
    mix = s1 / (s1 + s2)
    r1, r2 = a["geom_solref"][g1], a["geom_solref"][g2]
    if r1[0] > 0 and r2[0] > 0:
        solref = mix * r1 + (1 - mix) * r2
    else:
        solref = np.minimum(r1, r2)
    solimp = mix * a["geom_solimp"][g1] + (1 - mix) * a["geom_solimp"][g2]
    fr = np.maximum(a["geom_friction"][g1], a["geom_friction"][g2])
    assert dim in (1, 3, 4)
    return np.array([margin, margin - gap, dim, fr[0], fr[1], solref[0], solref[1], *solimp], dtype=np.float64)
