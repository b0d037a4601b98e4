"""Time final observations (`final_obs=True`): the step with and without them, and the final-observation kernel alone.

Workloads (bench.py's, fused random policy): c2 and c3 at 8 192 envs, c5 at 2 048 (snapshot reset), each with staggered
episodes (replica e starts at t = e*T/E, so about E/T replicas finish per step) and with lock-step episodes (every replica
finishes in the same step, once per T steps).  Arms, alternated in one process:
  off   env.step() of an env made without final_obs (the default);
  on    env.step() of an env made with final_obs=True: the step, then aie_observe_final (one CTA of four warps per env).
Reported per workload and regime: ms per step of each arm (CUDA events over --steps steps, or over whole episodes in the
lock-step regime, --rounds rounds, median and range); the final-observation kernel alone with the done flags
of a step in which about E/T replicas finished (staggered), every replica finished (lock-step) and none finished - 50
launches back to back behind a long device sleep, so that the host's enqueue time is not in the window - and the host
time of one observe_final() call; and the stand-alone observation pass (aie_observe) for scale.  The card's name, power
limit and maximum SM clock are printed with the numbers.

    python tools/time_final_obs.py [--steps 300] [--rounds 5] [--workloads c2,c3,c5] [--obs-dtype float32] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.time_obs_dtype import WORKLOADS, card, events_ms  # noqa: E402


def kernel_ms(torch, fn, n=50):
    """Device time per launch of fn, n launches back to back: a device sleep is enqueued first and outlasts the host's
    enqueueing, so the events bracket the kernels alone.  Also returns the host time of one call (enqueue only)."""
    import time
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    torch.cuda._sleep(50_000_000)   # ~25 ms at 2 GHz
    ev[0].record()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    host = (time.perf_counter() - t0) / n
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / n, 1e3 * host


def make(torch, key, final_obs, lockstep, obs_dtype):
    from ai_economist_b200 import foundation, workloads as wl
    cfg, E, reset = WORKLOADS[key]
    name, kw = wl.product_kwargs(cfg)
    if reset:
        kw["device_reset"] = reset
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seeds=[1000 + e for e in range(E)],
                                       auto_reset=True, final_obs=final_obs, obs_dtype=obs_dtype, **kw)
    env.reset()
    st = env.stepper
    T = int(env.episode_length)
    if not lockstep:
        st.state_view("t").copy_((torch.arange(E, device="cuda:0", dtype=torch.int64) * T // E).to(torch.int32))
    st.set_fused_policy(1234)
    return env


def run(torch, key, steps, rounds, lockstep, obs_dtype):
    envs = {"off": make(torch, key, False, lockstep, obs_dtype), "on": make(torch, key, True, lockstep, obs_dtype)}
    T = int(envs["off"].episode_length)
    for env in envs.values():   # one untimed episode, as bench.py
        for _ in range(T):
            env.stepper.step()
    torch.cuda.synchronize()
    n = T if lockstep else steps   # lock-step: whole episodes, one all-done step each
    ms = {k: [] for k in envs}
    for _ in range(rounds):
        for k, env in envs.items():
            ms[k].append(events_ms(torch, env.stepper.step, n))
    kernel = {}
    for k in [a for a in envs if a != "off"]:
        st, kk = envs[k].stepper, {}
        if lockstep:   # the env is at the start of an episode: step to its end, then to the step after it
            for _ in range(T):
                st.step()
            torch.cuda.synchronize()
            assert bool(st.buf["done"].all())
            kk["all_done"], kk["host"] = kernel_ms(torch, st.observe_final)
            st.step()
            torch.cuda.synchronize()
            assert not bool(st.buf["done"].any())
            kk["none_done"], _ = kernel_ms(torch, st.observe_final)
        else:
            st.step()
            kk["finished"] = int(st.buf["done"].sum())
            kk["some_done"], kk["host"] = kernel_ms(torch, st.observe_final)
        kernel[k] = {a: (round(v, 4) if isinstance(v, float) else v) for a, v in kk.items()}
    res = dict(workload=key, envs=envs["off"].n_envs, regime="lockstep" if lockstep else "staggered", obs_dtype=obs_dtype,
               steps_per_round=n, rounds=rounds, arms={}, final_kernel_ms=kernel,
               observe_only_ms=round(kernel_ms(torch, envs["on"].stepper.observe)[0], 4))
    for k in envs:
        v = sorted(ms[k])
        res["arms"][k] = dict(ms_per_step=round(v[len(v) // 2], 4), ms_range=[round(v[0], 4), round(v[-1], 4)])
    del envs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", default="c2,c3,c5")
    ap.add_argument("--regimes", default="staggered,lockstep")
    ap.add_argument("--obs-dtype", default="float32", choices=["float32", "bfloat16"])
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_final_obs.py needs a CUDA device")
    gpu = card() or torch.cuda.get_device_name(0)
    lines = []
    for key in args.workloads.split(","):
        for regime in args.regimes.split(","):
            r = run(torch, key, args.steps, args.rounds, regime == "lockstep", args.obs_dtype)
            r["gpu"] = gpu
            lines.append(json.dumps(r))
            print(lines[-1], flush=True)
            a = r["arms"]["off"]
            for k, b in r["arms"].items():
                print("  %-3s %-9s %s %-6s %.4f ms/step (%.4f-%.4f)  %+.1f %%  final kernel / host ms %s" % (
                    key, r["regime"], r["obs_dtype"], k, b["ms_per_step"], b["ms_range"][0], b["ms_range"][1],
                    100.0 * (b["ms_per_step"] / a["ms_per_step"] - 1.0), r["final_kernel_ms"].get(k, "")), flush=True)
            print("  %-3s %-9s observe-only %.4f ms" % (key, r["regime"], r["observe_only_ms"]), flush=True)
    print("card (name, power limit, max SM clock):", gpu)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
