"""metaworld_b200.post.StepPost against scalar transcriptions of the reference wrappers it vectorises
(metaworld/wrappers.py:35-88 RNNBasedMetaRLWrapper, :233-258 NormalizeRewardsExponential; stacking order and
RecordEpisodeStatistics placement from metaworld/__init__.py:437-446), and against its recorded outputs
(tests/golden/post_steppost.npz) on numpy and on torch inputs."""
import numpy as np
import pytest

from metaworld_b200.post import StepPost


class ScalarStack:
    """one sub-env's wrapper stack, written the way the reference applies it to a single env"""

    def __init__(self, recurrent, norm_in_obs, exponential, alpha):
        self.recurrent, self.norm_in_obs, self.exponential, self.alpha = recurrent, norm_in_obs, exponential, alpha
        self.mean, self.var, self.ep_ret = 0.0, 1.0, 0.0

    def reset(self, obs):
        self.ep_ret = 0.0
        return np.concatenate([obs, np.zeros(4), [0.0], [0.0]]) if self.recurrent else obs

    def _upd(self, r):
        self.mean = (1 - self.alpha) * self.mean + self.alpha * r
        self.var = (1 - self.alpha) * self.var + self.alpha * np.square(r - self.mean)

    def step(self, next_obs, action, reward, term, trunc):
        o = next_obs
        if self.recurrent:
            o = np.concatenate([next_obs, action, [float(reward) / 10.0 if self.norm_in_obs else float(reward)], [float(term or trunc)]])
        r = reward
        if self.exponential:
            self._upd(reward)          # step(): explicit update ...
            self._upd(reward)          # ... and a second one inside _apply_normalize_reward
            r = reward / (np.sqrt(self.var) + 1e-8)
        self.ep_ret += r
        return o, r


def test_steppost_matches_scalar_wrappers():
    rng = np.random.default_rng(0)
    N, D = 6, 49
    for recurrent, norm_in_obs, expo in [(True, True, True), (True, False, False), (False, True, True), (False, False, False)]:
        post = StepPost(N, recurrent, norm_in_obs, "exponential" if expo else None, reward_alpha=0.05)
        stacks = [ScalarStack(recurrent, norm_in_obs, expo, 0.05) for _ in range(N)]
        obs0 = rng.normal(size=(N, D))
        out = post.on_reset(obs0)
        ref = np.stack([s.reset(obs0[i]) for i, s in enumerate(stacks)])
        assert np.array_equal(out, ref)
        for t in range(40):
            term_obs, reset_obs = rng.normal(size=(N, D)), rng.normal(size=(N, D))
            act, rew = rng.uniform(-1, 1, size=(N, 4)), rng.normal(size=N) * 3
            term, trunc = rng.random(N) < 0.1, rng.random(N) < 0.1
            done = term | trunc
            obs_in = np.where(done[:, None], reset_obs, term_obs)                       # SAME_STEP autoreset: obs is the reset obs
            o, r, fo, fin = post.on_step(obs_in, act, rew, term, trunc, final_obs=term_obs)
            for i, s in enumerate(stacks):
                so, sr = s.step(term_obs[i], act[i], rew[i], term[i], trunc[i])
                assert np.isclose(r[i], sr, rtol=0, atol=1e-12)
                if done[i]:
                    assert np.allclose(fo[i], so) and np.isclose(fin[i], s.ep_ret)
                    assert np.allclose(o[i], s.reset(reset_obs[i]))
                else:
                    assert np.allclose(o[i], so) and fin[i] == 0.0


def _goldens():
    """tests/golden/post_steppost.npz and the generator that wrote it (its configurations and input replay)"""
    import importlib.util
    import os
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    spec = importlib.util.spec_from_file_location("make_post_goldens", os.path.join(here, "make_post_goldens.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    z = np.load(os.path.join(here, "post_steppost.npz"))
    return gen, z, {k[3:]: z[k] for k in z.files if k.startswith("in/")}


GEN, GOLD, INPUTS = _goldens()


@pytest.mark.parametrize("cfg", GEN.CONFIGS, ids=[GEN.config_name(*c) for c in GEN.CONFIGS])
def test_numpy_inputs_match_goldens(cfg):
    """The host path (`step` / `reset`) is bit-identical to the outputs recorded for every option combination."""
    out = GEN.run(GEN.make_post(*cfg), INPUTS, cfg[-1])
    for k, v in out.items():
        g = GOLD[f"{GEN.config_name(*cfg)}/{k}"]
        assert v.dtype == g.dtype and np.array_equal(v, g), k


@pytest.mark.parametrize("cfg", GEN.CONFIGS, ids=[GEN.config_name(*c) for c in GEN.CONFIGS])
def test_torch_inputs_match_goldens(cfg):
    """The same arithmetic on CPU tensors (what `step_torch` runs on the device): only torch's CPU `sqrt`, which is not
    correctly rounded, separates it from the goldens."""
    import torch
    post = GEN.make_post(*cfg)
    out = GEN.run(post, INPUTS, cfg[-1], convert=torch.from_numpy, back=lambda t: t.numpy())
    assert isinstance(post.ep_return, torch.Tensor)           # the state moved to torch and stayed there
    for k, v in out.items():
        np.testing.assert_allclose(v, GOLD[f"{GEN.config_name(*cfg)}/{k}"], rtol=1e-6, atol=0, err_msg=k)
