"""A/B of the separating-axis hints (mw_collide.cuh sep_hint_test) on one GPU: the standard build (B) against one
compiled with -DMW_NO_SEPCACHE (A).  Records the card (name, power limit, max SM clock), then runs bench.py on the two
builds alternately, A B A B A B for MT50 and A B once each for MT10 and ML45-train, and prints for every run ms_per_step,
the GJK/EPA share of own-work cycles, GJK/EPA cycles, convex pairs and GJK iterations per env step.  The outputs every
pair of runs dumped (--dump-outputs) are compared byte for byte.  Last, scripts/gpu_ab.py runs on both builds (MT50 @ 4096,
150 steps): equal per-step digests, and the hint counters of its profiled pass (tests and rejections).
Usage (on a GPU):  python scripts/gpu_sepcache_ab.py OUTDIR"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from metaworld_b200 import build as B  # noqa: E402

OUT = os.path.abspath(sys.argv[1])
os.makedirs(OUT, exist_ok=True)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True, timeout=60).stdout.strip()
print("card:", card, flush=True)
LIBS = {"A": B.build_variant(os.path.join(ROOT, "tests", "_build", "libmwb200_nosep.so"), ["MW_NO_SEPCACHE"]), "B": B.build()}


def run(cmd, lib):
    env = dict(os.environ, MW_B200_LIB=lib)
    env.pop("MW_B200_SPLIT_FRAC", None)
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    if r.returncode != 0:
        sys.exit(f"failed: {' '.join(cmd)}\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}")
    return r.stdout


def bench(build, benchmark, tag):
    dump = os.path.join(OUT, f"dump_{tag}")
    out = run([sys.executable, "bench.py", "--gpus", "1", "--steps", "100", "--warmup", "5", "--benchmark", benchmark,
               "--dump-outputs", dump, "--cpu-steps-per-env", "20"], LIBS[build])
    line = json.loads([x for x in out.splitlines() if x.startswith("{")][-1])
    ph = line["phases"]
    row = dict(build=build, benchmark=benchmark, tag=tag, ms_per_step=line["ms_per_step"], gjk_epa=ph["gjk_epa"],
               gjk_epa_cycles_per_env_step=ph["gjk_epa"] * ph["warp_cycles_per_env_step_own_work"],
               own_cycles_per_env_step=ph["warp_cycles_per_env_step_own_work"],
               convex_pairs_per_env_step=ph["convex_pairs_per_env_step"], gjk_iters_per_env_step=ph["gjk_iters_per_env_step"],
               contacts_dropped=line["solver"]["contacts_dropped"], clocks=line["clocks"], dump=dump)
    print(json.dumps(row), flush=True)
    return row


def same_dumps(a, b):
    names = sorted(os.listdir(a))
    return names == sorted(os.listdir(b)) and all(open(os.path.join(a, n), "rb").read() == open(os.path.join(b, n), "rb").read()
                                                   for n in names)


rows = []
for i in range(3):
    for build in "AB":
        rows.append(bench(build, "MT50", f"MT50_{build}{i}"))
for bm in ("MT10", "ML45-train"):
    for build in "AB":
        rows.append(bench(build, bm, f"{bm}_{build}"))
identical = {}
for bm in ("MT50", "MT10", "ML45-train"):
    r = [x for x in rows if x["benchmark"] == bm]
    identical[bm] = all(same_dumps(r[0]["dump"], x["dump"]) for x in r[1:])

ab = {}
for build in "AB":
    path = os.path.join(OUT, f"gpu_ab_{build}.json")
    run([sys.executable, os.path.join("scripts", "gpu_ab.py"), path, "150"], LIBS[build])
    ab[build] = json.load(open(path))
prof = ab["B"]["profile"]
summary = dict(card=card, rows=rows, outputs_identical=identical,
               gpu_ab=dict(steps_identical=ab["A"]["steps"] == ab["B"]["steps"], state_identical=ab["A"]["state"] == ab["B"]["state"],
                           dropped=[ab["A"]["dropped"], ab["B"]["dropped"]], profile_A=ab["A"]["profile"], profile_B=prof,
                           hint_tested_per_convex_pair=prof["n_sep_tested"] / max(1, prof["n_convex_pairs"]),
                           hint_rejected_per_convex_pair=prof["n_sep_rejected"] / max(1, prof["n_convex_pairs"])))
for bm in ("MT50", "MT10", "ML45-train"):
    for build in "AB":
        ms = [x["ms_per_step"] for x in rows if x["benchmark"] == bm and x["build"] == build]
        print(f"{bm:11s} {build}: ms_per_step {' '.join(f'{v:.4f}' for v in ms)}  spread {max(ms) - min(ms):.4f}")
print(json.dumps({k: v for k, v in summary.items() if k != "rows"}))
json.dump(summary, open(os.path.join(OUT, "sepcache_ab.json"), "w"), indent=1)
