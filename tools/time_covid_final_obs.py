"""Time COVID-19 final observations (`final_obs=True`): the c4 workload with the option off and on.

Workload: bench.py's c4 (4 096 envs, 540-step episodes, the device's random policy before every step).  Every replica
ends its episode on the same step, once per 540 steps.  Arms, alternated in one process for --rounds rounds, each round
one whole episode per arm:
  off   aie_covid_step (aie_covid_step_kernel), the default;
  on    aie_covid_step_final (aie_covid_step_final_kernel): the same step, and on the ending step the observation pass
        of the state the episode ended in, before the auto-reset.
Reported per arm (median over rounds, and range): ms per step over the whole episode (CUDA events around the episode,
sampler included); the step kernel's time on the episode-ending step; and its mean time on the 539 ordinary steps
(CUDA events around each step launch).  A device sleep is enqueued before each episode, so the host's enqueue runs
ahead and stays out of the windows.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/time_covid_final_obs.py [--rounds 5] [--envs 4096] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.time_obs_dtype import card  # noqa: E402


def make(E, final_obs):
    from ai_economist_b200 import foundation
    from ai_economist_b200.workloads import covid_reference_config
    cfg = covid_reference_config()
    env = foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=E, device="cuda:0", auto_reset=True,
                                       final_obs=final_obs, **cfg)
    env.reset()
    return env


def episode(torch, st, T, seed):
    """One whole episode from its first step: (ms per step, ending step's kernel ms, mean ordinary step kernel ms)."""
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
        raise SystemExit("time_covid_final_obs.py needs a CUDA device")
    gpu = card() or torch.cuda.get_device_name(0)
    envs = {"off": make(args.envs, False), "on": make(args.envs, True)}
    T = int(envs["off"].episode_length)
    for env in envs.values():   # one untimed episode per arm; each arm then starts every round at an episode's start
        episode(torch, env.stepper, T, 7)
    res = {k: [] for k in envs}
    for _ in range(args.rounds):
        for k, env in envs.items():
            res[k].append(episode(torch, env.stepper, T, 7))
    out = dict(workload="c4", envs=args.envs, episode_length=T, rounds=args.rounds, gpu=gpu, arms={})
    fields = ("ms_per_step", "end_step_kernel_ms", "ordinary_step_kernel_ms")
    for k, rows in res.items():
        arm = {}
        for j, f in enumerate(fields):
            v = sorted(r[j] for r in rows)
            arm[f] = dict(median=round(v[len(v) // 2], 5), range=[round(v[0], 5), round(v[-1], 5)])
        out["arms"][k] = arm
    line = json.dumps(out)
    print(line)
    off = out["arms"]["off"]
    print("%-4s %-26s %-26s %-26s" % ("arm", *fields))
    for k, arm in out["arms"].items():
        cells = []
        for f in fields:
            m, (lo, hi) = arm[f]["median"], arm[f]["range"]
            cells.append("%.4f (%.4f-%.4f) %+.1f%%" % (m, lo, hi, 100.0 * (m / off[f]["median"] - 1.0)))
        print("%-4s %-26s %-26s %-26s" % (k, *cells))
    print("card (name, power limit, max SM clock):", gpu)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
