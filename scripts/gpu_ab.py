"""A/B check of two builds or run-time switches of the engine: N random-action steps of a benchmark (MT50 @ 4096 by
default), per-step digests of obs / reward / info, the final device state (its bytes, `state`, and its values with
-0.0 read as +0.0, `state_values`), the step time, dropped contacts and the event counters of 20 profiled steps.  Usage (on a GPU):
  MW_B200_LIB=$PWD/tests/_build/libmwb200_no_sepcache.so python scripts/gpu_ab.py a.json
  python scripts/gpu_ab.py b.json
  python scripts/gpu_ab.py --cmp a.json b.json
Options --steps, --benchmark, --envs (150, MT50, 4096), or positionally: OUT [STEPS [BENCHMARK [ENVS]]].
From Python, `run_digests` does the first two in a child process."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SWITCHES = ("MW_B200_LIB", "MW_B200_SPLIT_FRAC")     # cleared for every run_digests child, then set as given


def run_digests(out, lib=None, switches=None, steps=150, benchmark="MT50", envs=4096):
    """Runs this script in a child process on the engine library `lib` (None: the standard build) with the run-time
    switches `switches` (environment variables, e.g. {"MW_B200_SPLIT_FRAC": "0.85"}) and returns the JSON it wrote to
    `out`."""
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    if lib:
        env["MW_B200_LIB"] = lib
    env.update(switches or {})
    cmd = [sys.executable, os.path.abspath(__file__), str(out), "--steps", str(steps), "--benchmark", benchmark, "--envs", str(envs)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    if r.returncode != 0:
        raise RuntimeError(f"{' '.join(cmd)} failed:\n{r.stdout}\n{r.stderr}")
    with open(out) as f:
        return json.load(f)


def compare(a_path, b_path):
    a, b = json.load(open(a_path)), json.load(open(b_path))
    bad = [i for i, (x, y) in enumerate(zip(a["steps"], b["steps"])) if x != y]
    print("A", a["build"]); print("B", b["build"])
    print("identical" if not bad and a["state"] == b["state"] else f"DIFFER first at step {bad[0] if bad else 'state only'} ({len(bad)} of {len(a['steps'])} steps)",
          "| ms/step A %.3f B %.3f" % (a["ms"], b["ms"]), "| dropped", a["dropped"], b["dropped"])


def digests(out, steps, benchmark, envs):
    import torch
    sys.path.insert(0, ROOT)
    from metaworld_b200.vector_env import make_mt_envs
    from metaworld_b200.engine import lib
    env = make_mt_envs(benchmark, seed=42, num_envs=envs, use_one_hot=True)
    env.reset(); env.enable_device_sampler()
    g = torch.Generator(device=env.device); g.manual_seed(3)
    step_digests = []
    for t in range(steps):
        a = torch.rand(envs, 4, device=env.device, generator=g) * 2 - 1
        o, r, te, tr, info = env.step_torch(a)
        h = hashlib.sha256(); h.update(o.cpu().numpy().tobytes()); h.update(r.cpu().numpy().tobytes()); h.update(info.cpu().numpy().tobytes())
        step_digests.append(h.hexdigest())
    torch.cuda.synchronize()
    st = env.engine.get_state()
    acts = [torch.rand(envs, 4, device=env.device, generator=g) * 2 - 1 for _ in range(60)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for a in acts:
        env.step_torch(a)
    e1.record(); torch.cuda.synchronize()
    dropped = env.engine.counters()["contacts_dropped"]
    env.engine.set_profiling(True); env.engine.profile()      # 20 profiled steps after everything compared: event counters (profile)
    for a in acts[:20]:
        env.step_torch(a)
    prof = env.engine.profile(); env.engine.set_profiling(False)
    with open(out, "w") as f:
        json.dump(dict(build=lib().mw_build_info().decode(), steps=step_digests, state=hashlib.sha256(st.tobytes()).hexdigest(),
                       state_values=hashlib.sha256(b"".join((st[k] + 0.0).tobytes() for k in st.dtype.names)).hexdigest(),
                       ms=e0.elapsed_time(e1) / len(acts), dropped=dropped, profile=prof), f)
    print("ok", out)


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("out", nargs="?", help="JSON file to write")
    # the positional form `OUT [STEPS [BENCHMARK [ENVS]]]` that existing callers use; the options take precedence
    p.add_argument("pos_steps", nargs="?", type=int, metavar="STEPS")
    p.add_argument("pos_benchmark", nargs="?", metavar="BENCHMARK")
    p.add_argument("pos_envs", nargs="?", type=int, metavar="ENVS")
    p.add_argument("--steps", type=int)
    p.add_argument("--benchmark")
    p.add_argument("--envs", type=int)
    p.add_argument("--cmp", nargs=2, metavar=("A", "B"), help="compare two JSON files written by earlier runs")
    args = p.parse_args(argv)
    if args.cmp:
        compare(*args.cmp)
    elif args.out:
        digests(args.out, args.steps or args.pos_steps or 150, args.benchmark or args.pos_benchmark or "MT50",
                args.envs or args.pos_envs or 4096)
    else:
        p.error("give OUT or --cmp A B")


if __name__ == "__main__":
    main()
