"""A/B check of two builds of the engine (MW_B200_LIB selects the library): MT50 @ 4096, N random-action steps, per-step
digests of obs / reward / info and the final device state.  Usage (on a GPU):
  MW_B200_LIB=$PWD/metaworld_b200/libmwb200_prev.so python scripts/gpu_ab.py a.json; python scripts/gpu_ab.py b.json; python scripts/gpu_ab.py --cmp a.json b.json"""
import hashlib, json, sys
if sys.argv[1] == "--cmp":
    a, b = json.load(open(sys.argv[2])), json.load(open(sys.argv[3]))
    bad = [i for i, (x, y) in enumerate(zip(a["steps"], b["steps"])) if x != y]
    print("A", a["build"]); print("B", b["build"])
    print("identical" if not bad and a["state"] == b["state"] else f"DIFFER first at step {bad[0] if bad else 'state only'} ({len(bad)} of {len(a['steps'])} steps)",
          "| ms/step A %.3f B %.3f" % (a["ms"], b["ms"]), "| dropped", a["dropped"], b["dropped"])
    sys.exit(0)
import numpy as np, torch
sys.path.insert(0, '.')
from metaworld_b200.vector_env import make_mt_envs
from metaworld_b200.engine import lib
BENCH = sys.argv[3] if len(sys.argv) > 3 else "MT50"
NENV = int(sys.argv[4]) if len(sys.argv) > 4 else 4096
env = make_mt_envs(BENCH, seed=42, num_envs=NENV, use_one_hot=True)
env.reset(); env.enable_device_sampler()
g = torch.Generator(device=env.device); g.manual_seed(3)
N = int(sys.argv[2]) if len(sys.argv) > 2 else 150
steps = []
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for t in range(N):
    a = torch.rand(NENV, 4, device=env.device, generator=g) * 2 - 1
    o, r, te, tr, info = env.step_torch(a)
    h = hashlib.sha256(); h.update(o.cpu().numpy().tobytes()); h.update(r.cpu().numpy().tobytes()); h.update(info.cpu().numpy().tobytes())
    steps.append(h.hexdigest())
torch.cuda.synchronize()
st = env.engine.get_state()
acts = [torch.rand(NENV, 4, device=env.device, generator=g) * 2 - 1 for _ in range(60)]
e0.record()
for a in acts:
    env.step_torch(a)
e1.record(); torch.cuda.synchronize()
N = 80
dropped = env.engine.counters()["contacts_dropped"]
env.engine.set_profiling(True); env.engine.profile()      # 20 profiled steps after everything compared: event counters (profile)
for a in acts[:20]:
    env.step_torch(a)
prof = env.engine.profile(); env.engine.set_profiling(False)
json.dump(dict(build=lib().mw_build_info().decode(), steps=steps, state=hashlib.sha256(st.tobytes()).hexdigest(), ms=e0.elapsed_time(e1) / (N - 20),
               dropped=dropped, profile=prof), open(sys.argv[1], "w"))
print("ok", sys.argv[1])
