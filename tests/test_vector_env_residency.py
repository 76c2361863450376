"""CPU suite: the vector env's numpy calls and their `_torch` twins share one last observation and one set of ended marks.
An env that replaces every other call of a fixed sequence with its torch twin returns what an all-numpy twin returns, in
every autoreset mode, with and without the optional wrappers.  Runs the REAL host code on the float64 oracle stand-in
(tests/oracle_engine.py).  The pseudorandom task selection never re-draws a task on reset, so no device sampler is
needed."""
import numpy as np
import pytest
import torch

from oracle_engine import oracle_vec_env

N = 20                                  # MT10 x 2 replicas
WRAPPERS = dict(normalize_observations=True, reward_normalization_method="gymnasium", recurrent_info_in_obs=True)


def _env(mode, wrappers):
    kw = WRAPPERS if wrappers else {}
    return oracle_vec_env("mt", "MT10", seed=4, num_goals=3, num_envs=N, max_episode_steps=4, task_select="pseudorandom",
                          autoreset_mode=mode, **kw)


def _host(x):
    return x.numpy().copy() if isinstance(x, torch.Tensor) else np.asarray(x).copy()


class _Driver:
    """Runs each call of the sequence in its numpy form, or in its torch form where `torch_form` says so, and returns
    what the call returned as numpy arrays.  A masked reset after a torch call takes the torch form: the numpy form needs
    the last observations on the host."""

    def __init__(self, env, torch_form):
        self.env, self.torch_form, self.k, self.last_torch = env, torch_form, 0, False

    def _use_torch(self, masked_reset=False):
        use = self.torch_form(self.k) or (masked_reset and self.last_torch)
        self.k += 1
        self.last_torch = use
        return use

    def reset(self):
        return [_host(self.env.reset_torch() if self._use_torch() else self.env.reset()[0])]

    def step(self, a):
        env = self.env
        if self._use_torch():
            obs, rew, term, trunc, _ = env.step_torch(torch.from_numpy(a))
        else:
            obs, rew, term, trunc, _ = env.step(a)
        out = [_host(obs), _host(rew).astype(np.float64), _host(term) != 0, _host(trunc) != 0]
        if env.autoreset_mode == "Disabled" and (out[2] | out[3]).any():     # restart the ended envs before the next step
            out += self.masked_reset(out[2] | out[3])
        return out

    def masked_reset(self, mask):
        if self._use_torch(masked_reset=True):
            return [_host(self.env.reset_torch(torch.from_numpy(mask)))]
        return [_host(self.env.reset(options={"reset_mask": mask})[0])]

    def save(self, mask):
        # numpy or torch mask; either way the call never synchronises
        return self.env.save_states(torch.from_numpy(mask) if self._use_torch() else mask)

    def load(self, states, mask):
        if self._use_torch():
            return [_host(self.env.load_states_torch(states, torch.from_numpy(mask)))]
        return [_host(self.env.load_states(states, mask))]

    def observe(self, mask):
        if self._use_torch():
            return [_host(self.env.observe_torch(torch.from_numpy(mask)))]
        return [_host(self.env.observe(mask))]

    def reset_goals(self, rv, mask, rv1):
        if self._use_torch():
            return [_host(self.env.reset_goals_torch(torch.from_numpy(rv), torch.from_numpy(mask), torch.from_numpy(rv1)))]
        return [_host(self.env.reset_goals(rv, mask, rv1))]


def _sequence(d, goals):
    rng = np.random.default_rng(0)
    acts = rng.uniform(-1, 1, size=(14, N, 4)).astype(np.float32)
    half, third = np.arange(N) % 2 == 0, np.arange(N) % 3 == 0
    out = d.reset()
    for a in acts[:3]:
        out += d.step(a)
    out += d.masked_reset(third)
    out += d.step(acts[3])
    states = d.save(np.ones(N, dtype=bool))
    for a in acts[4:7]:
        out += d.step(a)
    out += d.load(states, half)
    out += d.step(acts[7])
    out += d.masked_reset(half)
    out += d.observe(third)
    out += d.reset_goals(*goals)
    for a in acts[8:14]:
        out += d.step(a)
    out += d.masked_reset(~half)
    return out


@pytest.mark.parametrize("parity", [0, 1])
@pytest.mark.parametrize("wrappers", [False, True])
@pytest.mark.parametrize("mode", ["SameStep", "NextStep", "Disabled"])
def test_torch_twins_return_what_the_numpy_calls_return(mode, wrappers, parity):
    """`parity`: the calls k with k % 2 == parity take their torch form, so every call does in one of the two runs.  With
    parity 0 a torch masked reset follows a numpy step; with the optional wrappers its unmasked rows must be that step's
    observations, not those of the torch call before it."""
    ours, twin = _env(mode, wrappers), _env(mode, wrappers)
    rv, rv1 = twin.sample_goals(np.random.default_rng(1), np.arange(N) % 4 == 1)
    goals = (rv, np.arange(N) % 4 == 1, rv1)
    want = _sequence(_Driver(twin, lambda k: False), goals)
    got = _sequence(_Driver(ours, lambda k: k % 2 == parity), goals)
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, i
        if wrappers:            # torch's CPU sqrt is not correctly rounded, numpy's is
            np.testing.assert_allclose(g, w, rtol=1e-6, atol=0, err_msg=str(i))
        else:
            assert np.array_equal(g, w), i
