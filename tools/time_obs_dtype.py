"""Time the step with float32 and with bfloat16 observations, in one process, arms alternated.

Workloads (bench.py's, staggered episodes, fused random policy): c2 and c3 at 8 192 envs, c5 at 2 048 (snapshot reset).
Arms:
  f32         env.step() with float32 observations (the default);
  f32+to_bf16 the same step followed by `.to(torch.bfloat16)` of every float observation / mask tensor - what a trainer
              that feeds a bfloat16 policy does today;
  bf16        env.step() of an env made with obs_dtype=torch.bfloat16: the step kernel writes bfloat16 itself.
Per arm: ms per step (CUDA events over --steps steps, --rounds rounds alternated, median and range), the step kernel alone
(events around each launch), the stand-alone observation pass (aie_observe) and the bytes of observations written per
step.  The card's name and power limit are printed with the numbers.

    python tools/time_obs_dtype.py [--steps 300] [--rounds 5] [--workloads c2,c3,c5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

WORKLOADS = {"c2": ("c1_tutorial", 8192, None), "c3": ("c3_paper_tax", 8192, None), "c5": ("c5_full", 2048, "snapshot")}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out


def make(torch, key, obs_dtype):
    from ai_economist_b200 import foundation, workloads as wl
    cfg, E, reset = WORKLOADS[key]
    name, kw = wl.product_kwargs(cfg)
    if reset:
        kw["device_reset"] = reset
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seeds=[1000 + e for e in range(E)], auto_reset=True,
                                       obs_dtype=obs_dtype, **kw)
    env.reset()
    st = env.stepper
    T = int(env.episode_length)
    st.state_view("t").copy_((torch.arange(E, device="cuda:0", dtype=torch.int64) * T // E).to(torch.int32))
    st.set_fused_policy(1234)
    return env


def float_obs(env):
    b = env.stepper.buf
    return [b[k] for k in b if (k.startswith("obs_") or k.startswith("mask_")) and b[k].is_floating_point()]


def events_ms(torch, fn, n):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(n):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / n


def per_launch_ms(torch, fn, n):
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(2)] for _ in range(n)]
    for i in range(n):
        evs[i][0].record()
        fn()
        evs[i][1].record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in evs)[n // 2]


def run(torch, key, steps, rounds):
    f32, b16 = make(torch, key, torch.float32), make(torch, key, torch.bfloat16)
    T = int(f32.episode_length)
    for env in (f32, b16):   # one untimed episode, as bench.py
        for _ in range(T):
            env.stepper.step()
    torch.cuda.synchronize()
    sink = []

    def step_f32():
        f32.stepper.step()

    def step_f32_convert():
        f32.stepper.step()
        sink[:] = [t.to(torch.bfloat16) for t in float_obs(f32)]

    arms = {"f32": step_f32, "f32+to_bf16": step_f32_convert, "bf16": b16.stepper.step}
    for fn in arms.values():   # warm every shape
        for _ in range(10):
            fn()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            ms[k].append(events_ms(torch, fn, steps))
    obs_bytes = {k: sum(t.numel() * t.element_size() for t in float_obs(env)) +
                 sum(b.numel() * b.element_size() for n, b in env.stepper.buf.items() if n in ("obs_agent_idx", "obs_planner_idx"))
                 for k, env in (("f32", f32), ("bf16", b16))}
    conv_bytes = sum(t.numel() * (t.element_size() + 2) for t in float_obs(f32))
    res = dict(workload=key, envs=f32.n_envs, steps_per_round=steps, rounds=rounds, arms={})
    for k in arms:
        env = b16 if k == "bf16" else f32
        v = sorted(ms[k])
        res["arms"][k] = dict(
            ms_per_step=round(v[len(v) // 2], 4), ms_range=[round(v[0], 4), round(v[-1], 4)],
            step_kernel_ms=round(per_launch_ms(torch, env.stepper.step, 50), 4),
            observe_only_ms=round(per_launch_ms(torch, env.stepper.observe, 50), 4),
            obs_bytes_per_step=obs_bytes["bf16" if k == "bf16" else "f32"] + (conv_bytes if k == "f32+to_bf16" else 0))
    del f32, b16, sink
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", default="c2,c3,c5")
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_obs_dtype.py needs a CUDA device")
    gpu = card() or torch.cuda.get_device_name(0)
    lines = []
    for key in args.workloads.split(","):
        r = run(torch, key, args.steps, args.rounds)
        r["gpu"] = gpu
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
        for k, a in r["arms"].items():
            print("  %-3s %-12s %.4f ms/step (%.4f-%.4f)  step kernel %.4f ms  observe-only %.4f ms  obs bytes/step %.1f MB" % (
                key, k, a["ms_per_step"], a["ms_range"][0], a["ms_range"][1], a["step_kernel_ms"], a["observe_only_ms"],
                a["obs_bytes_per_step"] / 1e6), flush=True)
    print("card (name, power limit, max SM clock):", gpu)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
