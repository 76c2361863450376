"""Vectorised equivalents of the two per-sub-env wrappers the reference stacks between the one-hot wrapper and the
episode-statistics wrapper (metaworld/__init__.py:437-444):

* `RNNBasedMetaRLWrapper` (metaworld/wrappers.py:35-88): obs <- [obs, action, reward (/10), done]; after a reset the three
  extra blocks are zero;
* `NormalizeRewardsExponential` (wrappers.py:233-258): per-env exponential running mean / variance of the reward; the
  reference updates the estimate twice per step (once in `step`, once more inside `_apply_normalize_reward`), which is
  reproduced here because it changes the numbers.

* `gymnasium.wrappers.NormalizeReward` (reward_normalization_method="gymnasium", metaworld/__init__.py:441-442): reward
  divided by the running standard deviation of the discounted return (gamma 0.99; the return is zeroed on termination
  only, and never on reset);
* `gymnasium.wrappers.NormalizeObservation` (normalize_observations=True, metaworld/__init__.py:445-446): per-sub-env
  running mean / variance (Welford merge of one-sample batches, initial count 1e-4) over every observation the wrapper
  sees, i.e. step observations AND reset observations; output float32.

Elementwise ops on [N, ...] arrays; `MetaWorldVecEnv` applies them to what the engine returns.  Because the reference puts
`RecordEpisodeStatistics` outside the reward normalisation, the episodic return it reports is the sum of NORMALISED
rewards; `ep_return` below tracks that.

The arithmetic is written once against a small array namespace: numpy for `step` / `reset`, torch for `step_torch` (on
the device, without host synchronisation).  The per-env state lives in the namespace of the last call and is copied,
exactly, when a call arrives in the other one.  The host path is not torch on CPU tensors because torch's CPU `sqrt` is
not correctly rounded and numpy's is."""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

_NUMPY = SimpleNamespace(f32=np.dtype(np.float32), f64=np.dtype(np.float64), where=np.where, sqrt=np.sqrt, maybe_any=np.any,
                         zeros=np.zeros, cast=lambda x, dtype: np.asarray(x, dtype=dtype),
                         cat=lambda xs: np.concatenate(xs, axis=1), take=lambda x: x.cpu().numpy())


def _torch_namespace(device):
    import torch
    return SimpleNamespace(f32=torch.float32, f64=torch.float64, where=torch.where, sqrt=torch.sqrt,
                           maybe_any=lambda x: True,    # finding out would synchronise with the device; the masked form is exact
                           zeros=lambda shape, dtype: torch.zeros(shape, dtype=dtype, device=device),
                           cast=lambda x, dtype: x.to(dtype), cat=lambda xs: torch.cat(xs, dim=1),
                           take=lambda x: torch.from_numpy(x).to(device))


class StepPost:
    GAMMA, EPS = 0.99, 1e-8          # gymnasium's defaults; the reference passes none
    _STATE = ("mean", "var", "ret_mean", "ret_var", "ret_count", "disc", "obs_mean", "obs_var", "obs_count", "ep_return")

    def __init__(self, num_envs, recurrent_info_in_obs=False, normalize_reward_in_recurrent_info=True,
                 reward_normalization_method=None, reward_alpha=0.001, normalize_observations=False, obs_dtype=np.float64,
                 same_step=True):
        """`obs_dtype`: the dtype of the observations `on_step` gets on the host; the observation statistics are kept in it
        (gymnasium's `RunningMeanStd(dtype=observation_space.dtype)`) whatever the dtype of a device observation.
        `same_step`: the autoreset mode is SAME_STEP (a finished env's `obs` row is its reset observation); otherwise
        (NEXT_STEP / DISABLED) it is the terminal one, and a restart is a row of `on_step(restart=...)` or `on_reset(mask=...)`."""
        if reward_normalization_method not in (None, "exponential", "gymnasium"):
            raise ValueError(f"unknown reward_normalization_method {reward_normalization_method!r}")
        self.n = num_envs
        self.recurrent = bool(recurrent_info_in_obs)
        self.norm_in_obs = bool(normalize_reward_in_recurrent_info)
        self.exponential = reward_normalization_method == "exponential"
        self.gym_reward = reward_normalization_method == "gymnasium"
        self.norm_obs = bool(normalize_observations)
        self.alpha = float(reward_alpha)
        self.extra = 6 if self.recurrent else 0
        self.obs_dtype = np.dtype(obs_dtype)
        self.same_step = bool(same_step)
        self.mean, self.var = np.zeros(num_envs), np.ones(num_envs)          # NormalizeRewardsExponential
        # NormalizeReward.return_rms and .discounted_reward of every sub-env
        self.ret_mean, self.ret_var, self.ret_count = np.zeros(num_envs), np.ones(num_envs), np.full(num_envs, 1e-4)
        self.disc = np.zeros(num_envs)
        self.obs_mean = self.obs_var = self.obs_count = None                # NormalizeObservation.obs_rms, shaped at the first call
        self.ep_return = np.zeros(num_envs)
        self.xp, self._torch = _NUMPY, None

    @property
    def active(self):
        return self.recurrent or self.exponential or self.gym_reward or self.norm_obs

    def _use(self, obs):
        """The namespace of `obs`; the state is copied there when the previous call used the other one."""
        if self.norm_obs and self.obs_mean is None:        # first call: the state is still in numpy
            shape = (self.n, obs.shape[1] + self.extra)
            self.obs_mean, self.obs_var = np.zeros(shape, self.obs_dtype), np.ones(shape, self.obs_dtype)
            self.obs_count = np.full((self.n, 1), 1e-4)
        if isinstance(obs, np.ndarray):
            xp = _NUMPY
        else:
            self._torch = self._torch or _torch_namespace(obs.device)
            xp = self._torch
        if xp is not self.xp:
            for k in self._STATE:
                if getattr(self, k) is not None:
                    setattr(self, k, xp.take(getattr(self, k)))
            self.xp = xp
        return xp

    def save_rows(self):
        """A copy of every env's wrapper state, in the namespace it is in now (`load_rows` takes it back)."""
        return {k: v.copy() if isinstance(v, np.ndarray) else v.clone() for k in self._STATE if (v := getattr(self, k)) is not None}

    def load_rows(self, rows, mask, src):
        """Env e's wrapper state becomes row `src[e]` of `rows` (a `save_rows` result) where `mask[e]`.  `mask` (bool [N]) and
        `src` (integer [N], in range) are numpy arrays or device tensors; the state moves to their namespace."""
        xp = self._use(mask)
        for k, v in rows.items():
            if isinstance(v, np.ndarray) != (xp is _NUMPY):
                v = xp.take(v)
            setattr(self, k, xp.where(mask if v.ndim == 1 else mask[:, None], v[src], getattr(self, k)))

    @staticmethod
    def _merge(xp, mean, var, count, x):
        """N independent copies of gymnasium's RunningMeanStd.update (wrappers/utils.py), each fed one sample: the
        parallel-variance merge with batch mean = x, batch variance = 0, batch count = 1.  Arithmetic runs in the dtype of
        `mean`, with the float64 count converted at each use, like a Python-float count combined with float32 arrays in the
        per-env wrapper.  -> (mean, var, count)"""
        tot = count + 1.0
        c, tt = xp.cast(count, mean.dtype), xp.cast(tot, mean.dtype)
        delta = x - mean
        return mean + delta / tt, (var * c + delta * delta * c / tt) / tt, tot

    def _normalize_obs(self, xp, obs, mask=None):
        """NormalizeObservation.observation on the rows selected by `mask` (all when None): update, then normalise."""
        x = xp.cast(obs, self.obs_mean.dtype)
        mean, var, count = self._merge(xp, self.obs_mean, self.obs_var, self.obs_count, x)
        if mask is not None:
            m = mask[:, None]
            mean, var, count = xp.where(m, mean, self.obs_mean), xp.where(m, var, self.obs_var), xp.where(m, count, self.obs_count)
        self.obs_mean, self.obs_var, self.obs_count = mean, var, count
        return xp.cast((x - mean) / xp.sqrt(var + self.EPS), xp.f32)

    def on_reset(self, obs, mask=None):
        """obs [N, D] -> [N, D + extra]; the reward statistics are NOT reset (the wrapper object lives across episodes).
        `mask` [N] bool: a partial reset (`reset_mask`); only those rows' state changes, and only those output rows mean
        anything."""
        xp = self._use(obs)
        self.ep_return = xp.zeros(self.n, xp.f64) if mask is None else xp.where(mask, 0.0, self.ep_return)
        if self.recurrent:
            obs = xp.cat([obs, xp.zeros((self.n, 6), obs.dtype)])
        if self.norm_obs:
            obs = self._normalize_obs(xp, obs, mask)
        return obs

    def on_step(self, obs, actions, reward, terminated, truncated, final_obs=None, restart=None):
        """Returns (obs_out, reward_out [float64], final_obs_out, episode_return_of_finished_envs).
        SAME_STEP: `obs` holds the post-autoreset observation for finished envs and `final_obs` their terminal one; it
        may be None when no env finished.  NEXT_STEP: `restart` [N] bool marks the envs this call restarted (their `obs` row
        is the reset observation, reward 0): they get the reset treatment - zero recurrent extension, observation statistics
        updated with the reset observation, reward statistics untouched, reward 0 - and the others the step treatment."""
        xp = self._use(obs)
        done = (terminated | truncated) != 0
        reward = xp.cast(reward, xp.f64)
        obs_out, final_out = obs, final_obs
        fresh = done if self.same_step else restart        # rows of `obs` that are reset observations (None: none)
        if self.recurrent:
            r_obs = reward / 10.0 if self.norm_in_obs else reward
            ext = xp.cat([xp.cast(actions, obs.dtype).reshape(self.n, 4), xp.cast(r_obs[:, None], obs.dtype),
                          xp.cast(done[:, None], obs.dtype)])
            if final_obs is not None:
                final_out = xp.cat([final_obs, ext])
            obs_out = xp.cat([obs, ext if fresh is None else xp.where(fresh[:, None], 0, ext)])   # a freshly reset env reports zeros
        reward_out = reward
        keep = (lambda new, old: new) if restart is None else (lambda new, old: xp.where(restart, old, new))
        if self.exponential:
            mean, var = self.mean, self.var
            for _ in range(2):          # the reference updates the estimate twice per step (wrappers.py:250-258)
                mean = (1 - self.alpha) * mean + self.alpha * reward
                d = reward - mean
                var = (1 - self.alpha) * var + self.alpha * (d * d)
            self.mean, self.var = keep(mean, self.mean), keep(var, self.var)
            reward_out = reward / (xp.sqrt(self.var) + 1e-8)
        elif self.gym_reward:
            disc = self.disc * self.GAMMA * (1.0 - xp.cast(terminated, xp.f64)) + reward
            ret_mean, ret_var, ret_count = self._merge(xp, self.ret_mean, self.ret_var, self.ret_count, disc)
            self.disc, self.ret_mean = keep(disc, self.disc), keep(ret_mean, self.ret_mean)
            self.ret_var, self.ret_count = keep(ret_var, self.ret_var), keep(ret_count, self.ret_count)
            reward_out = reward / xp.sqrt(self.ret_var + self.EPS)
        if restart is not None:
            reward_out = xp.where(restart, 0.0, reward_out)
        if self.norm_obs:
            # the wrapper sees the step observation of every env (the terminal one for a finished env), then - SAME_STEP -
            # the reset observation of the finished ones: two updates for those, in that order.  The second one is masked,
            # so it leaves the other envs' statistics as they were; the host skips it when no env finished
            if self.same_step and final_out is not None and xp.maybe_any(done):
                normed = self._normalize_obs(xp, xp.where(done[:, None], final_out, obs_out))
                obs_out = xp.where(done[:, None], self._normalize_obs(xp, obs_out, done), normed)
                final_out = normed
            else:
                obs_out = self._normalize_obs(xp, obs_out)
        self.ep_return = self.ep_return + reward_out
        finished = xp.where(done, self.ep_return, 0.0)
        self.ep_return = xp.where(done, 0.0, self.ep_return)
        return obs_out, reward_out, final_out, finished
