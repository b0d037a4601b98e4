"""Time COVID-19 bfloat16 observations (`obs_dtype=torch.bfloat16`): the c4 workload in three arms, each with
`final_obs` off and on.

Workload: bench.py's c4 (4 096 envs, 540-step episodes, the device's random policy before every step).  Every replica
ends its episode on the same step, once per 540 steps.  Arms, alternated in one process for --rounds rounds, each round
one whole episode per arm:
  f32       the float32 step (aie_covid_step_kernel / aie_covid_step_final_kernel), the default;
  f32+conv  the same step, then what a bfloat16 trainer runs after it without the option: `.to(torch.bfloat16)` of the
            seven observation / mask tensors (and of their final_ twins with final_obs);
  bf16      the bfloat16 step (aie_covid_step_bf16_kernel / aie_covid_step_final_bf16_kernel).
Reported per arm (median over rounds, and range): ms per step over the whole episode (CUDA events around the episode,
sampler included); the time of the episode-ending step; and the mean time of the 539 ordinary steps (CUDA events
around each step launch and, in f32+conv, its conversion).  A device sleep is enqueued before each episode, so the
host's enqueue runs ahead and stays out of the windows.  The card's name, power limit and maximum SM clock are read
in the same run.

    python tools/time_covid_obs_dtype.py [--rounds 5] [--envs 4096] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.time_obs_dtype import card  # noqa: E402

OBS = ["obs_agent_state", "obs_postsubsidy", "obs_lagged_stringency", "obs_policy_indicators", "obs_scalars",
       "mask_agent", "mask_planner"]


def make(E, obs_dtype, final_obs):
    from ai_economist_b200 import foundation
    from ai_economist_b200.workloads import covid_reference_config
    cfg = covid_reference_config()
    env = foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=E, device="cuda:0", auto_reset=True,
                                       obs_dtype=obs_dtype, final_obs=final_obs, **cfg)
    env.reset()
    return env


def episode(torch, st, T, seed, convert):
    """One whole episode from its first step: (ms per step, ending step ms, mean ordinary step ms).  convert: the
    buffers a trainer converts to bfloat16 after each step."""
    E = torch.cuda.Event
    whole = [E(enable_timing=True) for _ in range(2)]
    per = [[E(enable_timing=True) for _ in range(2)] for _ in range(T)]
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)   # ~50 ms at 2 GHz: the host enqueues the episode while the device sleeps
    whole[0].record()
    for i in range(T):
        st.sample_random_actions(seed=seed)
        per[i][0].record()
        st.step()
        for b in convert:
            b.to(torch.bfloat16)
        per[i][1].record()
    whole[1].record()
    torch.cuda.synchronize()
    assert bool(st.buf["done"].all()), "the timed window must end on the episode's last step"
    k = [a.elapsed_time(b) for a, b in per]
    return whole[0].elapsed_time(whole[1]) / T, k[-1], sum(k[:-1]) / (T - 1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_covid_obs_dtype.py needs a CUDA device")
    gpu = card() or torch.cuda.get_device_name(0)
    arms = {}   # name -> (env, buffers converted after each step)
    for fo in (False, True):
        sfx = "/final" if fo else ""
        f32 = make(args.envs, torch.float32, fo)
        names = OBS + (["final_" + k for k in OBS] if fo else [])
        arms["f32" + sfx] = (f32, [])
        conv = make(args.envs, torch.float32, fo)
        arms["f32+conv" + sfx] = (conv, [conv.stepper.buf[k] for k in names])
        arms["bf16" + sfx] = (make(args.envs, torch.bfloat16, fo), [])
    T = int(arms["f32"][0].episode_length)
    for env, conv in arms.values():   # one untimed episode per arm; each arm then starts every round at an episode's start
        episode(torch, env.stepper, T, 7, conv)
    res = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, (env, conv) in arms.items():
            res[k].append(episode(torch, env.stepper, T, 7, conv))
    out = dict(workload="c4", envs=args.envs, episode_length=T, rounds=args.rounds, gpu=gpu, arms={})
    fields = ("ms_per_step", "end_step_ms", "ordinary_step_ms")
    for k, rows in res.items():
        arm = {}
        for j, f in enumerate(fields):
            v = sorted(r[j] for r in rows)
            arm[f] = dict(median=round(v[len(v) // 2], 5), range=[round(v[0], 5), round(v[-1], 5)])
        out["arms"][k] = arm
    line = json.dumps(out)
    print(line)
    print("%-15s %-30s %-30s %-30s" % ("arm (vs f32)", *fields))
    for k, arm in out["arms"].items():
        base = out["arms"]["f32/final" if k.endswith("/final") else "f32"]
        cells = []
        for f in fields:
            m, (lo, hi) = arm[f]["median"], arm[f]["range"]
            cells.append("%.4f (%.4f-%.4f) %+.1f%%" % (m, lo, hi, 100.0 * (m / base[f]["median"] - 1.0)))
        print("%-15s %-30s %-30s %-30s" % (k, *cells))
    print("card (name, power limit, max SM clock):", gpu)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
