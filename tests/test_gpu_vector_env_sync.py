"""GPU suite (-m gpu): the vector env's `_torch` calls and `save_states` never synchronise with the host, in every
autoreset mode, with and without the optional wrappers."""
import numpy as np
import pytest

from rig import torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

WRAPPERS = dict(normalize_observations=True, reward_normalization_method="gymnasium", recurrent_info_in_obs=True)


@pytest.mark.parametrize("wrappers", [False, True])
@pytest.mark.parametrize("mode", ["SameStep", "NextStep", "Disabled"])
def test_torch_surface_does_not_synchronise(torch_cuda, mode, wrappers):
    """MT10 @ 200 with short episodes: every torch entry point runs once to warm up (first uses allocate buffers, upload
    tables, start the device sampler and build the float64 env table), then twice under
    torch.cuda.set_sync_debug_mode("error").  No call leaves a fault."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    n = 200
    env = make_mt_envs("MT10", seed=1, num_envs=n, max_episode_steps=5, autoreset_mode=mode, **(WRAPPERS if wrappers else {}))
    dev = env.device
    rng = np.random.default_rng(0)
    acts = [torch.from_numpy(rng.uniform(-1, 1, size=(n, 4)).astype(np.float32)).to(dev) for _ in range(3)]
    mask = torch.arange(n, device=dev) % 3 == 0
    src = torch.roll(torch.arange(n, device=dev), 10)           # env e takes env e - 10's state: the same task type
    rv, rv1 = (torch.from_numpy(x).to(dev) for x in env.sample_goals(np.random.default_rng(3)))
    env.reset_torch()

    def surface(a):
        _, _, term, trunc, _ = env.step_torch(a)
        if mode == "Disabled":
            env.reset_torch((term | trunc) != 0)
        env.reset_torch(mask)
        qpos, qvel = env.get_state_torch()
        env.set_state_torch(qpos, qvel, mask)
        env.observe_torch(mask)
        env.query_torch(mask, bodies=("hand",), touching=True)
        env.expert_actions_torch()
        env.save_states(mask)
        states = env.save_states()
        env.load_states_torch(states, mask, src)
        env.reset_goals_torch(rv, mask, rv1)

    surface(acts[0])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for a in acts[1:]:
            surface(a)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert not env.engine.faults().any()
    env.close()
