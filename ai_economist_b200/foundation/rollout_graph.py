"""A bound rollout recorded once as a CUDA graph and replayed (`env.capture_rollout(act)`), shared by the
gather-trade-build and COVID-19 batched envs.

The library keeps the bookkeeping (include/aie_b200.h, aie_rollout_capture_begin): during the capture the policy sampler
reads its call counter on the device and the COVID-19 step finds its final row on the device, and after each replay the
host-side counters advance by what the captured calls did.  This module adds what only Python knows: the env's slot
views, the warm-up before the capture, and the refusal of every env call inside `act` but sample_actions."""


class RolloutGraph:
    """T iterations of `act(t, rollout.obs_slots[t])` then `env.step(env.action_buffers)`, recorded by
    env.capture_rollout().  replay() runs them again from cursor 0 and leaves the cursor at T."""

    def __init__(self, env, graph, generation):
        self._env, self._graph, self._generation = env, graph, generation

    @property
    def valid(self):
        """False once the rollout was unbound or re-bound, a checkpoint was loaded, reset() was tried mid-rollout, or
        another rollout was captured in this env."""
        return self._env._graph_generation == self._generation

    def replay(self):
        env = self._env
        if not self.valid:
            raise ValueError("replay: this graph no longer matches the env (the rollout was unbound or re-bound, a "
                             "checkpoint was loaded, reset() was tried mid-rollout or another rollout was captured); "
                             "capture it again")
        st = env._stepper
        if st.rollout_slot != 0:
            raise ValueError("replay: the bound rollout is at slot %d; a replay starts at slot 0 (after reset() or "
                             "restart_rollout())" % st.rollout_slot)
        st.rollout_replay_begin()
        self._graph.replay()
        st.rollout_replay_end()
        env._aim_rollout()


def invalidate(env):
    """Every RolloutGraph of env stops replaying (ValueError)."""
    env._graph_generation = getattr(env, "_graph_generation", 0) + 1


def refuse_in_act(env, fn):
    if getattr(env, "_in_capture_act", False):
        raise ValueError("%s: not available inside capture_rollout's act, which may call sample_actions only" % fn)


def capture_rollout(env, act):
    """env.capture_rollout(act): see BatchedFoundationEnv.capture_rollout."""
    refuse_in_act(env, "capture_rollout")
    st, r = env._stepper, env._rollout
    if not getattr(st, "supports_rollout_capture", False):
        raise NotImplementedError("this env's stepper cannot capture rollouts (the CUDA stepper can)")
    if r is None:
        raise ValueError("capture_rollout: no rollout bound (bind_rollout(T) first)")
    if not env._loaded:
        raise ValueError("capture_rollout: reset() first")
    if st.rollout_slot != 0:
        raise ValueError("capture_rollout: the bound rollout is at slot %d; capture at slot 0 (after reset() or "
                         "restart_rollout())" % st.rollout_slot)
    import torch

    dev = st.device
    # torch's warm-up before a capture, at slot 0 on a side stream; its draws are given back (counters), and so are the
    # slot's actions it overwrote.  What act writes elsewhere is the caller's, and the first replay overwrites it.
    counters = st.get_counters()
    actions0 = [a.clone() for a in r.actions[0]]
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    try:
        with torch.cuda.stream(side):
            _call_act(env, act, 0, r.obs_slots[0])
    finally:
        torch.cuda.current_stream(dev).wait_stream(side)
        for a, a0 in zip(r.actions[0], actions0):
            a.copy_(a0)
        st.set_counters(counters)
    invalidate(env)   # the library keeps one capture per handle: an earlier graph's deltas are gone
    g = torch.cuda.CUDAGraph()
    st.rollout_capture_begin()
    try:
        with torch.cuda.device(dev), torch.cuda.graph(g):
            for t in range(r.T):
                _call_act(env, act, t, r.obs_slots[t])
                env.step(env.action_buffers)
    finally:
        st.rollout_capture_end()
        env._aim_rollout()
    return RolloutGraph(env, g, env._graph_generation)


def _call_act(env, act, t, obs):
    env._in_capture_act = True
    try:
        act(t, obs)
    finally:
        env._in_capture_act = False
