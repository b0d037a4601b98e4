"""Time the evaluation of stored actions (`env.evaluate_actions` + backward) against the torch code a trainer writes
without it.

Workloads: c2 and c3 at 8 192 envs, c5 at 2 048 (snapshot reset), COVID-19 (c4) at 4 096; staggered episodes (replica
e starts at t = e*T/E) and one untimed episode first, as bench.py.  A rollout of --rollout steps stores the masks, the
actions sample_actions drew and its float32 logits (finite, so that no segment has an all -inf softmax); the minibatch is
--minibatch rows of those T*E stored steps, gathered and made contiguous.  Per call, both arms compute
loss = sum(log_prob) + 0.01 * sum(entropy) over every segment from leaf logits and run loss.backward():
  torch   per segment: masked_fill(mask == 0, -inf), log_softmax, gather at the stored action, the entropy, then
          autograd.  Equal-size segments are batched (single-action agents, planner brackets, COVID states);
          multi-action subspaces are one slice each.
  ours    env.evaluate_actions(...): one forward launch, one backward launch (--per-unit shapes are timed too for the
          GTB workloads: AIE_POLICY_PER_UNIT 0 one warp per row, 1 one warp per (row, unit)).
Reported per workload: device time per call (forward + backward; calls back to back behind a device sleep, so host
enqueue time is outside the window) of each arm, alternated over --rounds rounds in one process (median and range), and
the GB/s implied by the shapes (both launches: logits, masks and actions read twice, log-probabilities and entropies
written, their upstream gradients read, the logits' gradient written).  The card's name, power limit and maximum SM
clock are printed with the numbers.

    python tools/time_evaluate_actions.py [--rounds 5] [--calls 20] [--workloads c2,c3,c5,c4] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.time_obs_dtype import card  # noqa: E402
from tools.time_policy_sampler import kernel_ms, make_covid, make_gtb  # noqa: E402

MINIBATCH = {"c2": 16384, "c3": 16384, "c5": 4096, "c4": 16384}   # rows of stored steps per minibatch


def rollout(torch, env, steps):
    """sample_actions + step for `steps` steps: stacked [T*E, ...] logits, actions and masks (contiguous)."""
    st = env.stepper
    aa_b, ap_b = env.action_buffers
    planner = st._policy_shapes()[1] is not None
    sa, sp = st._policy_shapes()[:2]
    g = torch.Generator(device="cuda:0").manual_seed(0)
    rec = {k: [] for k in ("la", "lp", "aa", "ap", "ma", "mp")}
    for _ in range(steps):
        la = torch.randn(sa, device="cuda:0", generator=g) * 2
        lp = torch.randn(sp, device="cuda:0", generator=g) * 2 if planner else None
        rec["ma"].append(st.buf["mask_agent"].clone())
        rec["mp"].append(st.buf["mask_planner"].clone() if planner else None)
        env.sample_actions(la, lp, seed=3)
        rec["la"].append(la)
        rec["lp"].append(lp)
        rec["aa"].append(aa_b.clone())
        rec["ap"].append(ap_b.clone() if planner else None)
        env.step(env.action_buffers)
    return {k: (None if v[0] is None else torch.cat(v)) for k, v in rec.items()}


def gtb_torch_arm(torch, env):
    """The torch evaluation of a gather-trade-build env: (la, lp, aa, ap, ma, mp) -> loss."""
    from ai_economist_b200 import workloads as wl
    spec, d = env.spec, env.stepper.dims
    multi = bool(spec["multi_action_agents"])
    seg_a = wl.mask_segments(spec, "a") if multi else [d.mask_agent]
    n_p = d.n_act_planner

    def seg(x, m, a):
        logp = torch.log_softmax(x.masked_fill(m == 0, float("-inf")), -1)
        lp = logp.gather(-1, a.long().unsqueeze(-1)).squeeze(-1)
        p = logp.exp()
        return lp.sum() + 0.01 * (-(p * logp.masked_fill(p == 0, 0.0)).sum())

    def loss(la, lp, aa, ap, ma, mp):
        out, off = 0.0, 0
        for si, n in enumerate(seg_a):
            out = out + seg(la[..., off:off + n], ma[..., off:off + n], aa[..., si])
            off += n
        if n_p:
            N = la.shape[0]
            out = out + seg(lp.view(N, n_p, -1), mp.view(N, n_p, -1), ap)
        return out

    return loss


def covid_torch_arm(torch, env):
    def seg(x, m, a):
        logp = torch.log_softmax(x.masked_fill(m == 0, float("-inf")), -1)
        lp = logp.gather(-1, a.long().unsqueeze(-1)).squeeze(-1)
        p = logp.exp()
        return lp.sum() + 0.01 * (-(p * logp.masked_fill(p == 0, 0.0)).sum())

    def loss(la, lp, aa, ap, ma, mp):
        return seg(la, ma.transpose(1, 2), aa) + seg(lp, mp, ap)

    return loss


def run(torch, key, rounds, calls, steps, rows):
    covid = key == "c4"
    env = make_covid(torch) if covid else make_gtb(torch, key)
    st = env.stepper
    for _ in range(int(env.episode_length)):   # one untimed episode (random actions from the device sampler)
        st.sample_random_actions(seed=7)
        st.step()
    R = rollout(torch, env, steps)
    total = R["la"].shape[0]
    pick = torch.randperm(total, device="cuda:0", generator=torch.Generator(device="cuda:0").manual_seed(1))[:rows]
    mb = {k: (None if v is None else v.index_select(0, pick).contiguous()) for k, v in R.items()}
    planner = mb["lp"] is not None
    la = mb["la"].requires_grad_(True)
    lp = mb["lp"].requires_grad_(True) if planner else None
    args = (mb["aa"], mb["ap"]), (mb["ma"], mb["mp"])
    arm_torch = (covid_torch_arm if covid else gtb_torch_arm)(torch, env)

    def reset_grads():
        la.grad = None
        if planner:
            lp.grad = None

    def ours():
        reset_grads()
        lpa, lpp, ha, hp = env.evaluate_actions(la, lp, *args)
        loss = lpa.sum() + 0.01 * ha.sum()
        if planner:
            loss = loss + lpp.sum() + 0.01 * hp.sum()
        loss.backward()

    def torch_arm():
        reset_grads()
        arm_torch(la, lp, mb["aa"], mb["ap"], mb["ma"], mb["mp"]).backward()

    # bytes from shapes, both launches: logits + masks + actions read twice, log-probs + entropies written, their
    # upstream gradients read, the logits' gradient written
    elems = la.numel() + (lp.numel() if planner else 0)
    melems = mb["ma"].numel() + (mb["mp"].numel() if planner else 0)
    slots = mb["aa"].numel() + (mb["ap"].numel() if planner else 0)
    nbytes = 2 * (4 * elems + mb["ma"].element_size() * melems + 4 * slots) + 16 * slots + 4 * elems
    arms = {"torch": torch_arm, "ours": ours}
    if not covid:
        for pu in ("0", "1"):
            arms["ours_per_unit_" + pu] = (lambda pu: lambda: (os.environ.__setitem__("AIE_POLICY_PER_UNIT", pu), ours()))(pu)
    times = {k: [] for k in arms}
    for fn in arms.values():   # warm-up (the autograd graph, the caching allocator)
        fn()
        os.environ.pop("AIE_POLICY_PER_UNIT", None)
    torch.cuda.synchronize()
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(kernel_ms(torch, fn, calls))
            os.environ.pop("AIE_POLICY_PER_UNIT", None)
    res = dict(workload=key, envs=env.n_envs, rows=rows, bytes_per_call=nbytes, ms_per_call={}, gbps={})
    for k, v in times.items():
        v = sorted(v)
        med = v[len(v) // 2]
        res["ms_per_call"][k] = dict(median=round(med, 4), range=[round(v[0], 4), round(v[-1], 4)])
        res["gbps"][k] = round(nbytes / med / 1e6, 1)
    del env, R, mb
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rollout", type=int, default=4, help="stored steps per replica the minibatch is drawn from")
    ap.add_argument("--workloads", default="c2,c3,c5,c4")
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_evaluate_actions.py needs a CUDA device")
    gpu = card() or torch.cuda.get_device_name(0)
    lines = []
    for key in args.workloads.split(","):
        r = run(torch, key, args.rounds, args.calls, args.rollout, MINIBATCH[key])
        r["gpu"] = gpu
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
        for k, v in r["ms_per_call"].items():
            print("  %-3s %-16s %.4f ms/call (%.4f-%.4f)  %7.1f GB/s" % (key, k, v["median"], v["range"][0], v["range"][1],
                                                                       r["gbps"][k]), flush=True)
    print("card (name, power limit, max SM clock):", gpu)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
