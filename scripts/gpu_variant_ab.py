"""A/B of a build variant on one GPU: the standard build (B) against one compiled with extra -D macros (A), e.g.
-D MW_SERIAL_LINKS (link-by-link kinematics) or -D MW_NO_SEPCACHE (no separating-axis hints).  Records the card (name,
power limit, max SM clock), then runs bench.py on the two builds alternately, A B N times for MT50 and once each for
MT10 and ML45-train, and prints for every run ms_per_step, the clocks bench.py read, its whole `phases` and `solver`
records, and the warp cycles per env step of every phase.  The outputs every pair of runs dumped (--dump-outputs) are
compared byte for byte.  Last, scripts/gpu_ab.py runs on both builds (MT50 @ 4096, 150 steps): equal per-step digests
and final device state, and both builds' event counters (`kin`, the sep-hint counters, ...).
Usage (on a GPU):  python scripts/gpu_variant_ab.py OUTDIR -D MACRO [-D MACRO ...] [--mt50-pairs N]"""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BENCHMARKS = ("MT50", "MT10", "ML45-train")


def run_bench(lib, benchmark, dump):
    env = dict(os.environ, MW_B200_LIB=lib)
    env.pop("MW_B200_SPLIT_FRAC", None)
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "100", "--warmup", "5", "--benchmark", benchmark,
           "--dump-outputs", dump, "--cpu-steps-per-env", "20"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    if r.returncode != 0:
        sys.exit(f"failed: {' '.join(cmd)}\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}")
    return json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])


def same_dumps(a, b):
    names = sorted(os.listdir(a))
    return names == sorted(os.listdir(b)) and all(open(os.path.join(a, n), "rb").read() == open(os.path.join(b, n), "rb").read()
                                                   for n in names)


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("outdir")
    p.add_argument("-D", dest="defines", action="append", required=True, metavar="MACRO", help="-D macro of the A build")
    p.add_argument("--mt50-pairs", type=int, default=2, help="A B pairs of MT50 runs")
    args = p.parse_args(argv)
    out = os.path.abspath(args.outdir)
    os.makedirs(out, exist_ok=True)

    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from builds import run_digests, variant_lib
    from gpu_timing_common import card
    from metaworld_b200 import build as B
    c = card()
    print("card:", c, flush=True)
    libs = {"A": variant_lib(*args.defines), "B": B.build()}

    rows = []
    plan = [("MT50", i) for i in range(args.mt50_pairs)] + [(bm, 0) for bm in BENCHMARKS[1:]]
    for bm, i in plan:
        for build in "AB":
            tag = f"{bm}_{build}{i}"
            line = run_bench(libs[build], bm, os.path.join(out, f"dump_{tag}"))
            ph = line["phases"]      # shares of own-work cycles, and per-env-step counts
            own = ph["warp_cycles_per_env_step_own_work"]
            row = dict(build=build, benchmark=bm, tag=tag, ms_per_step=line["ms_per_step"], clocks=line["clocks"], phases=ph,
                       solver=line["solver"],
                       cycles_per_env_step={k: v * own for k, v in ph.items() if k != "unit" and "per_env_step" not in k},
                       dump=os.path.join(out, f"dump_{tag}"))
            print(json.dumps(row), flush=True)
            rows.append(row)
    identical = {}
    for bm in BENCHMARKS:
        r = [x for x in rows if x["benchmark"] == bm]
        identical[bm] = all(same_dumps(r[0]["dump"], x["dump"]) for x in r[1:])

    ab = {b: run_digests(os.path.join(out, f"gpu_ab_{b}.json"), libs[b]) for b in "AB"}
    summary = dict(card=c, defines=args.defines, rows=rows, outputs_identical=identical,
                   gpu_ab=dict(steps_identical=ab["A"]["steps"] == ab["B"]["steps"], state_identical=ab["A"]["state"] == ab["B"]["state"],
                               dropped=[ab["A"]["dropped"], ab["B"]["dropped"]], build_A=ab["A"]["build"], build_B=ab["B"]["build"],
                               profile_A=ab["A"]["profile"], profile_B=ab["B"]["profile"]))
    for bm in BENCHMARKS:
        for build in "AB":
            ms = [x["ms_per_step"] for x in rows if x["benchmark"] == bm and x["build"] == build]
            print(f"{bm:11s} {build}: ms_per_step {' '.join(f'{v:.4f}' for v in ms)}  spread {max(ms) - min(ms):.4f}")
    print(json.dumps({k: v for k, v in summary.items() if k != "rows"}))
    with open(os.path.join(out, "variant_ab.json"), "w") as f:
        json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
