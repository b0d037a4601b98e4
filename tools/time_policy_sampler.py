"""Time the policy sampler (`env.sample_actions`) against the torch code a trainer writes without it.

Workloads: c2 and c3 at 8 192 envs, c5 at 2 048 (snapshot reset), COVID-19 (c4) at 4 096; staggered episodes (replica e
starts at t = e*T/E) and one untimed episode first, as bench.py.  Fixed float32 logits of the masks' shape (finite, so
that no segment has an all -inf softmax).  Arms, alternated in one process:
  torch   per segment: masked_fill(mask == 0, -inf), Categorical(logits=...).sample() and .log_prob() (validate_args off:
          no host synchronisation), then an int32 copy into env.action_buffers.  Equal-size segments are batched into one
          Categorical (single-action agents, planner brackets, COVID); multi-action subspaces are one call each.
  ours    env.sample_actions(logits_agent, logits_planner, seed=...): one launch (--per-unit forces either launch shape
          of the GTB kernel: 0 one warp per env, 1 one warp per (env, unit)).
Reported per workload: device time per call of each arm (launches back to back behind a device sleep, so host enqueue time
is outside the window), achieved GB/s from bytes computed from shapes (logits + masks read, actions + log-probs written),
and ms per step of the whole `sample + step` loop (CUDA events over --steps steps, --rounds rounds, median and range).
For the GTB workloads `ours` is also timed with each launch shape (per_unit 0 / 1).  The card's name, power limit and
maximum SM clock are printed with the numbers.

    python tools/time_policy_sampler.py [--steps 200] [--rounds 5] [--workloads c2,c3,c5,c4] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.time_obs_dtype import WORKLOADS, card, events_ms  # noqa: E402


def kernel_ms(torch, fn, n):
    """Device time per call of fn, n calls back to back behind a device sleep that outlasts the host's enqueueing."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)   # ~50 ms at 2 GHz
    ev[0].record()
    for _ in range(n):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / n


def make_gtb(torch, key):
    from ai_economist_b200 import foundation, workloads as wl
    cfg, E, reset = WORKLOADS[key]
    name, kw = wl.product_kwargs(cfg)
    if reset:
        kw["device_reset"] = reset
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seeds=[1000 + e for e in range(E)],
                                       auto_reset=True, **kw)
    env.reset()
    T = int(env.episode_length)
    env.stepper.state_view("t").copy_((torch.arange(E, device="cuda:0", dtype=torch.int64) * T // E).to(torch.int32))
    return env


def make_covid(torch, E=4096):
    from ai_economist_b200 import foundation
    from ai_economist_b200.workloads import covid_reference_config
    cfg = covid_reference_config()
    name = cfg.pop("scenario_name")
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", auto_reset=True, **cfg)
    env.reset()
    T = int(env.episode_length)
    env.stepper.buf["hdr"][:, 0] = (torch.arange(E, device="cuda:0") * T // E).to(torch.int32)
    return env


def gtb_torch_arm(torch, env):
    """The torch sampler of a gather-trade-build env: a closure (logits_agent, logits_planner) -> (log-probs)."""
    from torch.distributions import Categorical
    from ai_economist_b200 import workloads as wl
    st, spec = env.stepper, env.spec
    aa, ap = env.action_buffers
    ma, mp = st.buf["mask_agent"], st.buf["mask_planner"]
    d = st.dims
    multi = bool(spec["multi_action_agents"])
    seg_a = wl.mask_segments(spec, "a") if multi else [d.mask_agent]
    n_p = d.n_act_planner

    def sample(la, lp):
        out, off = [], 0
        for si, n in enumerate(seg_a):
            dist = Categorical(logits=la[..., off:off + n].masked_fill(ma[..., off:off + n] == 0, float("-inf")),
                               validate_args=False)
            a = dist.sample()
            out.append(dist.log_prob(a))
            aa[..., si].copy_(a)
            off += n
        if n_p:
            E = la.shape[0]
            lg = lp.view(E, n_p, -1).masked_fill(mp.view(E, n_p, -1) == 0, float("-inf"))
            dist = Categorical(logits=lg, validate_args=False)
            a = dist.sample()
            out.append(dist.log_prob(a))
            ap.copy_(a)
        return out

    return sample


def covid_torch_arm(torch, env):
    from torch.distributions import Categorical
    st = env.stepper
    aa, ap = env.action_buffers
    ma, mp = st.buf["mask_agent"], st.buf["mask_planner"]

    def sample(la, lp):
        dist = Categorical(logits=la.masked_fill(ma.transpose(1, 2) == 0, float("-inf")), validate_args=False)
        a = dist.sample()
        aa.copy_(a)
        distp = Categorical(logits=lp.masked_fill(mp == 0, float("-inf")), validate_args=False)
        b = distp.sample()
        ap.copy_(b)
        return dist.log_prob(a), distp.log_prob(b)

    return sample


def run(torch, key, steps, rounds):
    covid = key == "c4"
    env = make_covid(torch) if covid else make_gtb(torch, key)
    st = env.stepper
    T = int(env.episode_length)
    for _ in range(T):   # one untimed episode (random actions from the device sampler)
        st.sample_random_actions(seed=7)
        st.step()
    torch.cuda.synchronize()
    E = env.n_envs
    g = torch.Generator(device="cuda:0").manual_seed(0)
    if covid:
        p = st.p
        sa, sp = (E, p["n_states"], 1 + p["num_stringency_levels"]), (E, 1 + p["num_subsidy_levels"])
        n_act = E * (p["n_states"] + 1)
        mask_elems, mask_bytes = E * (p["n_states"] * sa[2] + sp[1]), 4
        arm_torch = covid_torch_arm(torch, env)
    else:
        d = st.dims
        sa = (E, env.n_agents, d.mask_agent)
        sp = (E, d.mask_planner) if d.n_act_planner else None
        n_act = E * (env.n_agents * d.n_act_agent + d.n_act_planner)
        mask_elems = E * (env.n_agents * d.mask_agent + (d.mask_planner if d.n_act_planner else 0))
        mask_bytes = st.buf["mask_agent"].element_size()
        arm_torch = gtb_torch_arm(torch, env)
    la = torch.randn(sa, device="cuda:0", generator=g) * 2
    lp = torch.randn(sp, device="cuda:0", generator=g) * 2 if sp else None
    # bytes from shapes: logits + masks read, actions (int32) + log-probs (float32) written
    nbytes = 4 * mask_elems + mask_bytes * mask_elems + 8 * n_act
    calls = {"n": 0}

    def ours():
        calls["n"] += 1
        env.sample_actions(la, lp, seed=11)

    def torch_arm():
        arm_torch(la, lp)

    arms = {"torch": torch_arm, "ours": ours}
    res = dict(workload=key, envs=E, bytes_per_call=nbytes, kernel_ms={}, gbps={}, loop={})
    for k, fn in arms.items():
        fn()
        ms = kernel_ms(torch, fn, 20 if k == "torch" else 100)
        res["kernel_ms"][k] = round(ms, 4)
        res["gbps"][k] = round(nbytes / ms / 1e6, 1)
    if not covid:   # the two launch shapes of the GTB kernel
        for pu in ("0", "1"):
            os.environ["AIE_POLICY_PER_UNIT"] = pu
            ms = kernel_ms(torch, ours, 100)
            res["kernel_ms"]["ours_per_unit_" + pu] = round(ms, 4)
            res["gbps"]["ours_per_unit_" + pu] = round(nbytes / ms / 1e6, 1)
        del os.environ["AIE_POLICY_PER_UNIT"]
    step_only = []
    loop = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            loop[k].append(events_ms(torch, lambda: (fn(), st.step()), steps))
        step_only.append(events_ms(torch, st.step, steps))
    for k, v in list(loop.items()) + [("step_only", step_only)]:
        v = sorted(v)
        res["loop"][k] = dict(ms_per_step=round(v[len(v) // 2], 4), ms_range=[round(v[0], 4), round(v[-1], 4)])
    del env, arm_torch
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", default="c2,c3,c5,c4")
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_policy_sampler.py needs a CUDA device")
    gpu = card() or torch.cuda.get_device_name(0)
    lines = []
    for key in args.workloads.split(","):
        r = run(torch, key, args.steps, args.rounds)
        r["gpu"] = gpu
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
        for k, v in r["kernel_ms"].items():
            print("  %-3s %-16s %.4f ms/call  %7.1f GB/s" % (key, k, v, r["gbps"][k]), flush=True)
        for k, v in r["loop"].items():
            print("  %-3s loop %-10s %.4f ms/step (%.4f-%.4f)" % (key, k, v["ms_per_step"], v["ms_range"][0], v["ms_range"][1]),
                  flush=True)
    print("card (name, power limit, max SM clock):", gpu)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
