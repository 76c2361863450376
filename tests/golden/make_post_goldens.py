"""Generates tests/golden/post_steppost.npz: what metaworld_b200.post.StepPost returns on numpy inputs, for every
combination of its options and both observation dtypes, over one seeded input sequence with random terminations and
truncations (40 steps of 5 envs, terminal observations always given).  The file holds the inputs as well; tests/test_post.py
replays them through `run` below, on numpy and on torch inputs.  Written from the implementation the tests pin:
    python tests/golden/make_post_goldens.py
Keys: `in/<name>` inputs (obs has one row per step plus the reset observation); `<config>/<name>` outputs, where
`final_obs` keeps the rows of the finished envs only (step-major order)."""
import itertools
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from metaworld_b200.post import StepPost  # noqa: E402

N, D, STEPS, ALPHA = 5, 5, 40, 0.05
CONFIGS = list(itertools.product((False, True), (False, True), (None, "exponential", "gymnasium"), (False, True),
                                 (np.float32, np.float64)))


def config_name(recurrent, norm_in_obs, method, norm_obs, dtype):
    return f"rec{int(recurrent)}_nio{int(norm_in_obs)}_{method or 'none'}_nobs{int(norm_obs)}_{np.dtype(dtype).name}"


def make_inputs(seed=0):
    rng = np.random.default_rng(seed)
    return {"obs": rng.normal(size=(STEPS + 1, N, D)), "final_obs": rng.normal(size=(STEPS, N, D)),
            "actions": rng.uniform(-1, 1, size=(STEPS, N, 4)).astype(np.float32), "reward": rng.normal(size=(STEPS, N)) * 3,
            "terminated": rng.random((STEPS, N)) < 0.1, "truncated": rng.random((STEPS, N)) < 0.1}


def run(post, inp, dtype, convert=lambda x: x, back=np.asarray):
    """Feeds the sequence to `post` (after `convert`, e.g. to torch tensors); returns the outputs as numpy arrays."""
    out = {"reset": back(post.on_reset(convert(inp["obs"][0].astype(dtype))))}
    steps = []
    for t in range(STEPS):
        o, r, fo, fin = post.on_step(convert(inp["obs"][t + 1].astype(dtype)), convert(inp["actions"][t]), convert(inp["reward"][t]),
                                     convert(inp["terminated"][t]), convert(inp["truncated"][t]),
                                     final_obs=convert(inp["final_obs"][t].astype(dtype)))
        done = inp["terminated"][t] | inp["truncated"][t]
        steps.append((back(o), back(r), back(fo)[done], back(fin)))
    for k, v in zip(("obs", "reward", "final_obs", "episode_return"), zip(*steps)):
        out[k] = np.concatenate(v) if k == "final_obs" else np.stack(v)
    return out


def make_post(recurrent, norm_in_obs, method, norm_obs, dtype):
    return StepPost(N, recurrent, norm_in_obs, method, ALPHA, norm_obs, obs_dtype=dtype)


if __name__ == "__main__":
    inp = make_inputs()
    arrays = {f"in/{k}": v for k, v in inp.items()}
    for cfg in CONFIGS:
        for k, v in run(make_post(*cfg), inp, cfg[-1]).items():
            arrays[f"{config_name(*cfg)}/{k}"] = v
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "post_steppost.npz")
    np.savez_compressed(path, **arrays)
    print(f"{len(CONFIGS)} configurations -> {path}")
