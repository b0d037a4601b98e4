"""Time `env.compute_advantages` (advantages and value targets of a stored rollout) against the textbook torch reverse
loop a trainer writes without it.

Workloads: c2 and c3 at 8 192 envs with T = 200, c5 at 2 048 (snapshot reset) with T = 150, COVID-19 (c4) at 4 096 with
T = 90 and T = 540; staggered episodes (replica e starts at t = e*T_episode/E).  A rollout of T steps of sample_actions +
step from random logits stores the rewards and dones the env wrote; values, last values and final values are random
float32.  Arms, alternated over --rounds rounds in one process (median and range):
  ours       env.compute_advantages(..., final_values=..., gamma=0.998, lam=0.98): device time per call, calls back to
             back behind a device sleep (host enqueue outside the window), and the GB/s of the bytes the shapes imply
             (rewards, values, dones, last values read, advantages and returns written, final values read at done rows)
             against the 3.35 TB/s of the H100 SXM data sheet;
  torch f32  the reverse loop over t (torch.where for the bootstrap, delta, the (1 - done) carry), for the agents and
  torch f64  the planner, in float32 and in float64 (inputs converted first): device events around one whole call, so the
             host's enqueue is inside the window, and the host enqueue time alone (perf_counter around the call, no
             synchronise) beside it;
  rollout    for context, the T steps of sample_actions + step the call follows (device events).
The card's name, power limit and maximum SM clock are printed with the numbers.

    python tools/time_advantages.py [--rounds 5] [--calls 50] [--workloads c2,c3,c5,c4,c4_long] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.time_obs_dtype import card, events_ms  # noqa: E402
from tools.time_policy_sampler import kernel_ms, make_covid, make_gtb  # noqa: E402

HORIZON = {"c2": 200, "c3": 200, "c5": 150, "c4": 90, "c4_long": 540}
HBM_TBPS = 3.35   # H100 SXM data sheet; not a measured peak
GAMMA, LAM = 0.998, 0.98


def rollout(torch, env, T, store):
    """T steps of sample_actions + step; with store, the stacked rewards ([T, E, A], [T, E]) and dones [T, E]."""
    st = env.stepper
    sa, sp = st._policy_shapes()[:2]
    A = sa[1]
    g = torch.Generator(device="cuda:0").manual_seed(1)
    ra, rp, d = [], [], []
    for _ in range(T):
        la = torch.randn(sa, device="cuda:0", generator=g)
        lp = torch.randn(sp, device="cuda:0", generator=g) if sp is not None else None
        env.sample_actions(la, lp, seed=5)
        env.step(env.action_buffers)
        if store:
            if "reward" in st.buf:
                ra.append(st.buf["reward"][:, :A].contiguous())
                rp.append(st.buf["reward"][:, A].contiguous())
            else:
                ra.append(env.rew["a"].clone())
                rp.append(env.rew["p"].clone())
            d.append(env.done["__all__"].clone())
    return (torch.stack(ra), torch.stack(rp), torch.stack(d)) if store else None


def torch_gae(torch, r, v, d, lv, f, dt):
    """The textbook reverse loop of one group in dtype dt: (adv, ret)."""
    r, v, lv, f = r.to(dt), v.to(dt), lv.to(dt), f.to(dt)
    done = (d != 0).view(d.shape + (1,) * (r.dim() - 2))
    notdone = (~done).to(dt)
    adv = torch.empty_like(r)
    last = torch.zeros_like(lv)
    T = r.shape[0]
    for t in reversed(range(T)):
        nv = lv if t == T - 1 else v[t + 1]
        nv = torch.where(done[t], f[t], nv)
        delta = r[t] + GAMMA * nv - v[t]
        last = delta + GAMMA * LAM * notdone[t] * last
        adv[t] = last
    return adv, adv + v


def run(torch, key, rounds, calls):
    T = HORIZON[key]
    env = make_covid(torch) if key.startswith("c4") else make_gtb(torch, key)
    rollout(torch, env, T, False)                          # warm-up (and staggered episodes well under way)
    ra, rp, d = rollout(torch, env, T, True)
    E, A = ra.shape[1], ra.shape[2]
    g = torch.Generator(device="cuda:0").manual_seed(2)
    rnd = lambda *s: torch.randn(s, device="cuda:0", generator=g)
    va, vp, lva, lvp, fa, fp = rnd(T, E, A), rnd(T, E), rnd(E, A), rnd(E), rnd(T, E, A), rnd(T, E)
    n_done = int((d != 0).sum())
    nbytes = (ra.numel() * ra.element_size() + rp.numel() * rp.element_size() + 4 * (va.numel() + vp.numel())
              + 4 * d.numel() + 4 * (lva.numel() + lvp.numel()) + 2 * 4 * (ra.numel() + rp.numel()) + 4 * n_done * (A + 1))

    def ours():
        return env.compute_advantages((ra, rp), (va, vp), d, (lva, lvp), (fa, fp), gamma=GAMMA, lam=LAM)

    def torch_arm(dt):
        a = torch_gae(torch, ra, va, d, lva, fa, dt)
        p = torch_gae(torch, rp, vp, d, lvp, fp, dt)
        return a[0], p[0], a[1], p[1]

    def host_and_device(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        h0 = time.perf_counter()
        fn()
        h1 = time.perf_counter()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), (h1 - h0) * 1e3

    out, t32, t64 = ours(), torch_arm(torch.float32), torch_arm(torch.float64)   # warm-up every shape
    err = max(float((x.double() - y).abs().max()) for x, y in zip(out, t64))
    res = {k: [] for k in ("ours", "torch_f32", "torch_f32_host", "torch_f64", "torch_f64_host", "rollout")}
    for _ in range(rounds):
        res["ours"].append(kernel_ms(torch, ours, calls))
        dev, host = host_and_device(lambda: torch_arm(torch.float32))
        res["torch_f32"].append(dev)
        res["torch_f32_host"].append(host)
        dev, host = host_and_device(lambda: torch_arm(torch.float64))
        res["torch_f64"].append(dev)
        res["torch_f64_host"].append(host)
        res["rollout"].append(events_ms(torch, lambda: rollout(torch, env, T, False), 1))
    med = {k: statistics.median(v) for k, v in res.items()}
    gbps = nbytes / (med["ours"] * 1e-3) / 1e9
    return {"workload": key, "E": E, "A": A, "T": T, "columns": E * A + E, "done_rows": n_done, "bytes": nbytes,
            "ms": med, "ms_range": {k: [min(v), max(v)] for k, v in res.items()}, "gbps": gbps,
            "share_of_hbm_datasheet": gbps / (HBM_TBPS * 1e3), "max_abs_diff_vs_torch_f64": err}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--workloads", default="c2,c3,c5,c4,c4_long")
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_advantages.py needs a CUDA device")
    gpu = card() or torch.cuda.get_device_name(0)
    lines = []
    for key in args.workloads.split(","):
        r = run(torch, key, args.rounds, args.calls)
        r["gpu"] = gpu
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
        m = r["ms"]
        print("  %-7s E=%d T=%d: ours %.4f ms (%.0f GB/s, %.1f%% of %.2f TB/s) | torch f32 %.3f ms (host enqueue %.3f) | "
              "torch f64 %.3f ms (host enqueue %.3f) | rollout %.2f ms" % (
                  key, r["E"], r["T"], m["ours"], r["gbps"], 100 * r["share_of_hbm_datasheet"], HBM_TBPS, m["torch_f32"],
                  m["torch_f32_host"], m["torch_f64"], m["torch_f64_host"], m["rollout"]), flush=True)
        torch.cuda.empty_cache()
    print("card (name, power limit, max SM clock):", gpu)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
