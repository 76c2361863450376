"""Debug tool (needs a GPU): device vs oracle, per task.
  python scripts/gpu_diag.py reset    TASK...        # post-reset obs / qpos / qvel differences per goal
  python scripts/gpu_diag.py open     TASK...        # first diverging step of the open-loop golden rollout + contact comparison there
  python scripts/gpu_diag.py cr       TASK...        # worst teacher-forced step on the policy trajectory + contact comparison there
  python scripts/gpu_diag.py first    TASK...        # first env step after reset, substep by substep, contact lists at each
  python scripts/gpu_diag.py tf       [TASK...] [-v] # teacher-forced summary per task along the policy trajectory (all golden
                                                     # tasks by default); -v: one row per step, details of steps beyond 1e-4
  python scripts/gpu_diag.py contacts TASK K T [NSUB] # env K at policy state T: contact lists and qacc, NSUB substeps
  python scripts/gpu_diag.py live     TASK [STEPS]   # 4 fresh goals: snapshots vs oracle resets, then open loop vs a live oracle
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from rig import GOLD, Rig, _tasks_with_goldens  # noqa: E402
from oracle.tasks import TASKS as OT  # noqa: E402
from oracle import mjphys as P  # noqa: E402

np.set_printoptions(precision=6, suppress=True, linewidth=250)


def big(a, b, tol=1e-5):
    d = np.abs(np.asarray(a, float) - np.asarray(b, float))
    idx = np.where(~(d < tol))[0]
    return ", ".join(f"[{i}] dev {a[i]:.6f} ora {b[i]:.6f}" for i in idx[:12])


def oracle_env(task, rv):
    oe = OT[task](); oe.set_task_vec(rv[:len(oe.random_reset_space()[0])], False); oe.reset()
    return oe


def step_mocap(rig, oe, k, mocap, action):
    """Both sides: the step's mocap update from `mocap` and the gripper control of `action`; returns the control."""
    mp = np.clip(mocap + np.clip(action[:3], -1, 1) * 0.01, oe.mocap_low, oe.mocap_high)
    st = rig.eng.get_state(); st[k]["mocap_pos"] = mp; rig.eng.set_state(st)
    oe.data.mocap_pos[0][:] = mp; oe.data.mocap_quat[0][:] = [1, 0, 1, 0]
    ctrl = (float(action[3]), -float(action[3])); oe.data.ctrl = ctrl
    return ctrl


def compare_substeps(rig, oe, k, ctrl, nsub, every):
    """Forward pass of env k against the oracle's, substep by substep: contact and constraint counts, solver iterations,
    qacc error.  The contact lists and qacc of both sides are printed at every substep (`every`), or else at the first
    substep whose qacc differs, which ends the comparison."""
    nq, nv = oe.model.nq, oe.model.nv
    for sub in range(nsub):
        con, qacc, meta = rig.eng.debug_forward(ctrl)
        P.mj_forward(oe.model, oe.data)
        qe = np.abs(qacc[k, :nv] - oe.data.qacc).max()
        print(f'  substep {sub}: dev ncon {int(meta[k,0])} nefc {int(meta[k,1])} it {int(meta[k,2])} | ora ncon {oe.data.ncon} nefc {oe.data.nefc} it {oe.data.solver_iter} | qacc err {qe:.3e}')
        differs = qe > 1e-2 * max(1.0, np.abs(oe.data.qacc).max()) or not np.isfinite(qe)
        if every or differs:
            oc = sorted([(c.geom1, c.geom2, c.dist, *c.pos, *list(c.frame)[:3], oe.data.efc_force[c.efc_address] if c.efc_address >= 0 else 0) for c in oe.data.contact])
            dc = sorted([(int(c[7]), int(c[8]), c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[9]) for c in con[k][: int(meta[k, 0])]])
            for x in dc: print('    dev', np.array(x))
            for x in oc: print('    ora', np.array(x))
            print('    dev qacc', qacc[k, :nv]); print('    ora qacc', oe.data.qacc)
        if differs and not every:
            st = rig.eng.get_state(); print('    dev qpos', st[k]["qpos"][:nq]); print('    ora qpos', oe.data.qpos)
            return
        rig.eng.debug_substeps(1, ctrl); P.mj_step(oe.model, oe.data, 1)
        if every:
            st = rig.eng.get_state(); print('    qpos err', big(st[k]['qpos'][:nq], oe.data.qpos, 1e-6))


def contacts_at(rig, task, rv, k, qpos, qvel, mocap, action, nsub=5, every=False):
    """Sets env k and an oracle env to the same state, applies the action's mocap / ctrl, compares substep by substep."""
    oe = oracle_env(task, rv)
    st = rig.eng.get_state()
    st[k]["qpos"][:len(qpos)] = qpos; st[k]["qvel"][:len(qvel)] = qvel; st[k]["warm"][:] = 0
    rig.eng.set_state(st)
    oe.data.qpos = qpos; oe.data.qvel = qvel; oe.data.qacc_warmstart = 0
    compare_substeps(rig, oe, k, step_mocap(rig, oe, k, mocap, action), nsub, every)


def do_first(task):
    """first env step after reset, substep by substep (device snapshot state vs oracle reset state)"""
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    rig = Rig(torch, task, g["rand_vec"]); rig.reset()
    k = 0
    st = rig.eng.get_state()
    nq, nv = g["reset_qpos"].shape[1], g["reset_qvel"].shape[1]
    oe = oracle_env(task, g["rand_vec"][k])
    print(f"{task}: reset state: qpos {big(st[k]['qpos'][:nq], oe.data.qpos, 1e-7)} | qvel {big(st[k]['qvel'][:nv], oe.data.qvel, 1e-6)} | warm {big(st[k]['warm'][:nv], oe.data.qacc_warmstart, 1e-4)} | mocap {big(st[k]['mocap_pos'], oe.data.mocap_pos[0], 1e-7)}")
    compare_substeps(rig, oe, k, step_mocap(rig, oe, k, oe.data.mocap_pos[0].copy(), g["actions"][k, 0]), 5, every=True)


def do_reset(task):
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    rig = Rig(torch, task, g["rand_vec"]); snaps = rig.eng.get_snapshots()
    nq, nv = g["reset_qpos"].shape[1], g["reset_qvel"].shape[1]
    for k in range(rig.n):
        print(f"{task} goal {k}: obs: {big(snaps[k]['obs'], g['reset_obs'][k])} | qpos: {big(snaps[k]['st']['qpos'][:nq], g['reset_qpos'][k])} | qvel: {big(snaps[k]['st']['qvel'][:nv], g['reset_qvel'][k], 1e-4)}")


def do_open(task):
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    rv = g["rand_vec"].astype(np.float32) if os.environ.get("MW_DIAG_RV32") else g["rand_vec"]     # (float32-rounded goals: the pre-0892805 behaviour)
    rig = Rig(torch, task, rv); rig.reset()
    for t in range(g["actions"].shape[1]):
        o, r, info, _, _ = rig.step(g["actions"][:, t])
        e = np.abs(o - g["obs"][:, t]).max(axis=1)
        print(f"   t {t} obs err per env {e} reward err {np.abs(r - g['reward'][:, t])}")
        if (e > 1e-4).any() or not np.isfinite(e).all():
            k = int(np.nanargmax(np.where(np.isfinite(e), e, 1e9)))
            print(f"{task}: open-loop first divergence at step {t} env {k}: {big(o[k], g['obs'][k, t], 1e-4)}")
            if t > 0:
                contacts_at(rig, task, g["rand_vec"][k], k, g["qpos"][k, t - 1], g["qvel"][k, t - 1], g["mocap"][k, t - 1], g["actions"][k, t])
            return
    print(f"{task}: open-loop clean")


def policy_rig(g, task):
    """The rig of the policy trajectory, one step in: like the tests, rewards that latch state on their first call latch here."""
    rig = Rig(torch, task, g["p_rand_vec"]); rig.reset()
    rig.step(g["p_actions"][:, 0])
    return rig


def do_cr(task):
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    rig = policy_rig(g, task)
    worst = (-1, 0, 0)
    for t in range(g["p_actions"].shape[1] - 1):
        rig.load_golden(g, t, "p_")
        o, r, info, _, _ = rig.step(g["p_actions"][:, t + 1])
        e = np.abs(o - g["p_obs"][:, t + 1]).max(axis=1)
        e = np.where(np.isfinite(e), e, 1e9)
        if e.max() > worst[0]:
            worst = (float(e.max()), t, int(e.argmax()))
    e, t, k = worst
    print(f"{task}: contact-rich worst step err {e:.3e} at t {t} env {k}")
    contacts_at(rig, task, g["p_rand_vec"][k], k, g["p_qpos"][k, t], g["p_qvel"][k, t], g["p_mocap"][k, t], g["p_actions"][k, t + 1])


def do_tf(task, verbose):
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    if "p_actions" not in g:
        print(f"{task}: no policy trajectory in the fixture")
        return
    rig = policy_rig(g, task)
    nq, nv = g["p_qpos"].shape[2], g["p_qvel"].shape[2]
    T = g["p_actions"].shape[1]
    wo = wr = wq = wv = 0; bad = 0
    for t in range(T - 1):
        rig.load_golden(g, t, "p_")
        o, r, info, _, _ = rig.step(g["p_actions"][:, t + 1])
        s2 = rig.eng.get_state()
        eo = np.abs(o - g["p_obs"][:, t + 1]).max(axis=1); er = np.abs(r - g["p_reward"][:, t + 1])
        eq = np.abs(s2["qpos"][:, :nq] - g["p_qpos"][:, t + 1]).max(axis=1); ev = np.abs(s2["qvel"][:, :nv] - g["p_qvel"][:, t + 1]).max(axis=1)
        wo, wr, wq, wv = max(wo, eo.max()), max(wr, er.max()), max(wq, eq.max()), max(wv, ev.max()); bad += eo.max() > 1e-4
        if verbose:
            flag = max(eo.max(), er.max()) > 1e-4
            print(t, 'obs', eo, 'rew', er, 'qpos', eq, 'qvel', ev, '  <<<' if flag else '')
            if flag:
                k = int(np.argmax(eo + er))
                print('   dev obs', o[k][:18]); print('   ora obs', g["p_obs"][k, t + 1][:18]); print('   rew', r[k], g["p_reward"][k, t + 1], 'info', info[k], g["p_info"][k, t + 1])
                print('   dq', s2["qpos"][k, :nq] - g["p_qpos"][k, t + 1]); print('   dv', s2["qvel"][k, :nv] - g["p_qvel"][k, t + 1])
    c = rig.eng.counters()
    print(f"{task:28s} obs {wo:.1e} rew {wr:.1e} qpos {wq:.1e} qvel {wv:.1e} bad_steps {bad}/{T-1} dropped {c['contacts_dropped']} iters/pass {c['solver_iters']/c['forward_passes']:.2f}", flush=True)


def do_contacts(task, k, t, nsub):
    """Env k at state t of the policy trajectory: contact lists and qacc of both sides at every substep."""
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    rig = Rig(torch, task, g["p_rand_vec"]); rig.reset()
    contacts_at(rig, task, g["p_rand_vec"][k], k, g["p_qpos"][k, t], g["p_qvel"][k, t], g["p_mocap"][k, t], g["p_actions"][k, t + 1],
                nsub, every=True)


def do_live(task, steps, K=4):
    """K fresh goals: device snapshots vs oracle resets, then `steps` random actions open loop against live oracle envs."""
    from metaworld_b200.engine import lib
    from metaworld_b200.tasks import TASKS
    print(lib().mw_build_info().decode())
    spec = TASKS[task]
    rvs = np.random.default_rng(0).uniform(spec.rand_low, spec.rand_high, size=(K, 6))
    rig = Rig(torch, task, rvs)
    snaps = rig.eng.get_snapshots()
    oenvs = []
    for k in range(K):
        oe = OT[task](); oe.set_task_vec(rvs[k], False)
        oobs, _ = oe.reset()
        oenvs.append(oe)
        nq, nv = oe.model.nq, oe.model.nv
        dq = np.abs(snaps[k]['st']['qpos'][:nq] - oe.data.qpos).max()
        dv = np.abs(snaps[k]['st']['qvel'][:nv] - oe.data.qvel).max()
        do = np.abs(snaps[k]['obs'] - oobs).max()
        print(f'snap {k}: dq {dq:.2e} dv {dv:.2e} dobs {do:.2e}')
        if k == 0:
            print(' dev qpos', snaps[k]['st']['qpos'][:nq]); print(' ora qpos', oe.data.qpos)
            print(' dev obs', snaps[k]['obs']); print(' ora obs', oobs)
    print('reset obs err', np.abs(rig.reset() - np.stack([s['obs'] for s in snaps])).max())
    arng = np.random.default_rng(1)
    for t in range(steps):
        a = arng.uniform(-1, 1, size=(K, 4)).astype(np.float32)
        o, r, _, _, _ = rig.step(a)
        eo, er = [], []
        for k in range(K):
            oo, rr, _, _, _ = oenvs[k].step(a[k])
            eo.append(np.abs(oo - o[k]).max()); er.append(abs(rr - r[k]))
        if t % 10 == 0 or t == steps - 1:
            print(t, 'obs err', np.max(eo), 'rew err', np.max(er), 'ncon/iters', rig.eng.counters())
    st = rig.eng.get_state()
    print('final dq', np.abs(st[0]['qpos'][:nq] - oenvs[0].data.qpos).max())


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = p.add_subparsers(dest="mode", required=True)
    for mode in ("reset", "open", "cr", "first"):
        sub.add_parser(mode).add_argument("tasks", nargs="+")
    tf = sub.add_parser("tf")
    tf.add_argument("tasks", nargs="*")
    tf.add_argument("-v", "--verbose", action="store_true")
    c = sub.add_parser("contacts")
    c.add_argument("task"); c.add_argument("k", type=int); c.add_argument("t", type=int); c.add_argument("nsub", type=int, nargs="?", default=1)
    live = sub.add_parser("live")
    live.add_argument("task"); live.add_argument("steps", type=int, nargs="?", default=100)
    args = p.parse_args(argv)
    if args.mode == "contacts":
        return do_contacts(args.task, args.k, args.t, args.nsub)
    if args.mode == "live":
        return do_live(args.task, args.steps)
    if args.mode == "tf":
        fn, tasks = (lambda task: do_tf(task, args.verbose)), args.tasks or _tasks_with_goldens()
    else:
        fn, tasks = dict(reset=do_reset, open=do_open, cr=do_cr, first=do_first)[args.mode], args.tasks
    for task in tasks:
        try:
            fn(task)
        except Exception as ex:  # keep going: this is a survey tool
            print(f"{task}: {args.mode} raised {ex!r}")


if __name__ == "__main__":
    main()
