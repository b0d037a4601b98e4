"""Times rollouts stored in place (env.bind_rollout) against the copy loop of INTEGRATION §7, on cuda:0.

Arms, alternated over rounds, each with the same small fixed policy and value nets (one linear layer per head over the
flat observations):
  copy   sample_actions, step, then copy observations, masks, actions, rewards and done into [T, E, ...] buffers and
         run the value net over env.final_obs every step;
  bound  sample_actions and step into the bound rollout; one value-net pass over the [K, E, ...] final slots per rollout;
  step   sample_actions and step alone (no storage, no value net).
The bound arm's per-rollout restart (slot T copied into slot 0) is inside its timed region.  c4 (COVID-19, 4 096
replicas) runs the same arms with its own heads.  Then, per gather-trade-build workload, compute_advantages over the
stored rollout: from the stored [T, E, A + 1] rewards (split inside, one copy per group) against pre-split rewards, and
[K, ...] final values (per_episode_end) against [T, ...].  Prints the card's name and power limit, the bytes the copy
arm moves per step (from the shapes), and per workload the median and range of ms per step and per rollout.

    python tools/time_rollout.py [--workloads c2,c3,c5,c4] [--T 16] [--rounds 5]
"""
import argparse
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai_economist_b200 import foundation  # noqa: E402
from ai_economist_b200._abi import COVID_OBS_NAMES as COVID_OBS  # noqa: E402
from ai_economist_b200.workloads import product_kwargs  # noqa: E402

WORKLOADS = {"c2": ("c1_tutorial", 8192), "c3": ("c3_paper_tax", 8192), "c5": ("c5_full", 2048), "c4": ("covid", 4096)}


class Nets:
    """Policy and value heads: one linear layer each over the agents' and the planner's flat observations."""

    def __init__(self, env):
        g = torch.Generator(device="cuda").manual_seed(0)
        ot = env.obs_tensors
        fa, fp = ot["obs_agent_flat"].shape[-1], ot["obs_planner_flat"].shape[-1]
        na, npl = ot["mask_agent"].shape[-1], ot["mask_planner"].shape[-1]
        w = lambda i, o: torch.randn(i, o, device="cuda", generator=g) * 0.01
        self.pa, self.pp, self.va, self.vp = w(fa, na), w(fp, npl), w(fa, 1), w(fp, 1)

    def logits(self, ot):
        return ((ot["obs_agent_flat"].float() @ self.pa).contiguous(), (ot["obs_planner_flat"].float() @ self.pp).contiguous())

    def values(self, ot):
        return (ot["obs_agent_flat"].float() @ self.va).squeeze(-1), (ot["obs_planner_flat"].float() @ self.vp).squeeze(-1)


class CovidNets:
    """The same heads for the COVID-19 env, over each state's agent_state column and the planner's scalars."""

    def __init__(self, env):
        g = torch.Generator(device="cuda").manual_seed(0)
        sa, sp, _, _ = env.stepper._policy_shapes()
        w = lambda i, o: torch.randn(i, o, device="cuda", generator=g) * 0.01
        self.pa, self.pp, self.va, self.vp = w(6, sa[-1]), w(4, sp[-1]), w(6, 1), w(4, 1)

    def logits(self, ot):
        return ((ot["obs_agent_state"].float().transpose(-1, -2) @ self.pa).contiguous(),
                (ot["obs_scalars"].float() @ self.pp).contiguous())

    def values(self, ot):
        return (ot["obs_agent_state"].float().transpose(-1, -2) @ self.va).squeeze(-1), (ot["obs_scalars"].float() @ self.vp).squeeze(-1)


def obs_tensors(env):
    """The observation / mask tensors the env shows now (slot s when a rollout is bound)."""
    if hasattr(env, "obs_tensors"):
        return env.obs_tensors
    r = env.rollout
    return r.obs_slots[env.stepper.rollout_slot] if r is not None else {k: env.stepper.buf[k] for k in COVID_OBS}


def final_tensors(env):
    if hasattr(env, "final_obs_tensors"):
        return env.final_obs_tensors
    return {k: env.stepper.buf["final_" + k] for k in COVID_OBS}


def make(cfg, E):
    if cfg == "covid":
        from ai_economist_b200.workloads import COVID_KWARGS, covid_reference_config
        kw = covid_reference_config(dict(COVID_KWARGS))
        return foundation.make_env_instance(kw.pop("scenario_name"), n_envs=E, device="cuda:0", final_obs=True, **kw)
    name, kw = product_kwargs(cfg)
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seed=1, final_obs=True, **kw)
    return env


def run_copy(env, nets, T, seed):
    ot = obs_tensors(env)
    bufs = {k: torch.empty((T,) + tuple(v.shape), dtype=v.dtype, device="cuda") for k, v in ot.items()}
    aa, ap = env.action_buffers
    act = (torch.empty((T,) + tuple(aa.shape), dtype=aa.dtype, device="cuda"),
           torch.empty((T,) + tuple(ap.shape), dtype=ap.dtype, device="cuda"))
    rews = [b for k, b in env.stepper.buf.items() if k.startswith("reward")]
    rew = [torch.empty((T,) + tuple(b.shape), dtype=b.dtype, device="cuda") for b in rews]
    done = torch.empty((T, env.n_envs), dtype=torch.int32, device="cuda")
    fv = []
    for t in range(T):
        for k, v in ot.items():
            bufs[k][t].copy_(v)
        env.sample_actions(*nets.logits(ot), seed=seed)
        act[0][t].copy_(aa)
        act[1][t].copy_(ap)
        env.step(env.action_buffers)
        for dst, src in zip(rew, rews):
            dst[t].copy_(src)
        done[t].copy_(env.stepper.buf["done"])
        fv.append(nets.values(final_tensors(env)))


def run_bound(env, nets, T, seed):
    if env.stepper.rollout_slot:
        env.restart_rollout()   # slot T -> slot 0: part of every rollout after the first
    for t in range(T):
        env.sample_actions(*nets.logits(obs_tensors(env)), seed=seed)
        env.step(env.action_buffers)
    nets.values(env.rollout.final_obs_tensors)


def run_step(env, nets, T, seed):
    for t in range(T):
        env.sample_actions(*nets.logits(obs_tensors(env)), seed=seed)
        env.step(env.action_buffers)


def copy_bytes(env):
    """Bytes the copy arm reads and writes per step: every observation / mask tensor, the actions, rewards and done, read
    once and written once."""
    st = env.stepper
    n = sum(v.numel() * v.element_size() for v in obs_tensors(env).values())
    n += sum(b.numel() * b.element_size() for b in env.action_buffers)
    n += sum(b.numel() * b.element_size() for k, b in st.buf.items() if k.startswith("reward")) + st.buf["done"].numel() * 4
    return 2 * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3,c5,c4")
    ap.add_argument("--T", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card:", q)
    for wl in a.workloads.split(","):
        cfg, E = WORKLOADS[wl]
        envs = {k: make(cfg, E) for k in ("copy", "bound", "step")}
        envs["bound"].bind_rollout(a.T, final_obs=True)
        for env in envs.values():
            env.reset()
        nets = CovidNets(envs["copy"]) if cfg == "covid" else Nets(envs["copy"])
        fns = {"copy": run_copy, "bound": run_bound, "step": run_step}
        times = {k: [] for k in fns}
        for rnd in range(a.rounds + 1):
            for k, fn in fns.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(envs[k], nets, a.T, rnd + 1)
                torch.cuda.synchronize()
                if rnd:   # round 0 warms every shape up
                    times[k].append((time.perf_counter() - t0) * 1e3)
        print("%s: E=%d T=%d K=%d, copy arm moves %.1f MB per step" % (wl, E, a.T, envs["bound"].rollout.K,
                                                                      copy_bytes(envs["copy"]) / 1e6))
        for k, v in times.items():
            v = sorted(v)
            med = v[len(v) // 2]
            print("  %-5s ms/step %.4f (%.4f-%.4f)  ms/rollout %.2f (%.2f-%.2f)"
                  % (k, med / a.T, v[0] / a.T, v[-1] / a.T, med, v[0], v[-1]))
        if cfg != "covid":
            time_advantages(envs["bound"], a.rounds)
        del envs
        torch.cuda.empty_cache()


def time_advantages(env, rounds, reps=20):
    """compute_advantages over the bound rollout (its T steps are stored): stored rewards (split inside) against
    pre-split ones, [K, ...] final values against [T, ...]."""
    r, E, A = env.rollout, env.n_envs, env.n_agents
    T, K = r.T, r.K
    g = torch.Generator(device="cuda").manual_seed(1)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    V, LV = (rnd(T, E, A), rnd(T, E)), (rnd(E, A), rnd(E))
    FK, FT = (rnd(K, E, A), rnd(K, E)), (rnd(T, E, A), rnd(T, E))
    rew = r.buf["reward"]
    split = (rew[..., :A].contiguous(), rew[..., A].contiguous())
    arms = {"stored rewards, [K] finals": lambda: env.compute_advantages(rew, V, r.buf["done"], LV, FK, gamma=0.99,
                                                                         lam=0.95, per_episode_end=True),
            "pre-split rewards, [K] finals": lambda: env.compute_advantages(split, V, r.buf["done"], LV, FK, gamma=0.99,
                                                                            lam=0.95, per_episode_end=True),
            "pre-split rewards, [T] finals": lambda: env.compute_advantages(split, V, r.buf["done"], LV, FT, gamma=0.99,
                                                                            lam=0.95)}
    times = {k: [] for k in arms}
    for i in range(rounds + 1):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
            if i:
                times[k].append((time.perf_counter() - t0) * 1e3 / reps)
    for k, v in times.items():
        v = sorted(v)
        print("  advantages (T=%d, K=%d) %-30s ms/call %.4f (%.4f-%.4f)" % (T, K, k, v[len(v) // 2], v[0], v[-1]))


if __name__ == "__main__":
    main()
