"""foundation-b200: a Hopper-native (H100) batched stepper for the AI Economist "Foundation" environments.

    from ai_economist_b200 import foundation
    env = foundation.make_env_instance("layout_from_file/simple_wood_and_stone", n_envs=8192, **reference_kwargs)
    obs = env.reset()
    obs, rew, done, info = env.step(actions)

The per-timestep hot path runs as hand-written sm_90a CUDA kernels behind the C-ABI in include/aie_b200.h.
There is no CPU fallback: constructing an env without the compiled library or without a CUDA device raises.
"""
__version__ = "0.1.0"
