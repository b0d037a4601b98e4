"""Time COVID-19 episode metrics (`episode_metrics=True`): the c4 workload with the option off and on.

Workload: bench.py's c4 (4 096 envs, 540-step episodes, the device's random policy before every step).  Arms,
alternated in one process for --rounds rounds, each round one whole episode per arm:
  off   aie_covid_step_kernel, the default;
  on    aie_covid_step_stats_kernel<float>: the same step, which also adds the step's values to the episode-metric
        accumulators (about 2 KB read and 2 KB written per replica and step) and copies them on the ending step.
Reported per arm (median over rounds, and range): ms per step over the whole episode (CUDA events around the episode,
sampler included), the step kernel's time on the episode-ending step and its mean on the 539 ordinary steps (CUDA
events around each step launch; tools/time_covid_final_obs.py's episode()).  Also the device time of one
metrics_tensor() call (aie_covid_metrics_kernel, [4096, 415] float64; median of 50 calls, each between its own events)
and of one previous_episode_metrics_tensor().  A device sleep is enqueued before each episode so the host's enqueue runs
ahead.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/time_covid_metrics.py [--rounds 5] [--envs 4096] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.time_covid_final_obs import episode  # noqa: E402  (ms per step, ending step kernel ms, ordinary step kernel ms)
from tools.time_obs_dtype import card  # noqa: E402


def make(E, episode_metrics):
    from ai_economist_b200 import foundation
    from ai_economist_b200.workloads import covid_reference_config
    cfg = covid_reference_config()
    env = foundation.make_env_instance(cfg.pop("scenario_name"), n_envs=E, device="cuda:0", auto_reset=True,
                                       episode_metrics=episode_metrics, **cfg)
    env.reset()
    return env


def call_ms(torch, fn, n=50):
    E = torch.cuda.Event
    ev = [[E(enable_timing=True) for _ in range(2)] for _ in range(n)]
    out = fn()
    torch.cuda.synchronize()
    torch.cuda._sleep(50_000_000)
    for a, b in ev:
        a.record()
        fn(out)
        b.record()
    torch.cuda.synchronize()
    v = sorted(a.elapsed_time(b) for a, b in ev)
    return dict(median=round(v[n // 2], 5), range=[round(v[0], 5), round(v[-1], 5)])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_covid_metrics.py needs a CUDA device")
    gpu = card() or torch.cuda.get_device_name(0)
    envs = {"off": make(args.envs, False), "on": make(args.envs, True)}
    T = int(envs["off"].episode_length)
    for env in envs.values():   # one untimed episode per arm; each arm then starts every round at an episode's start
        episode(torch, env.stepper, T, 7)
    res = {k: [] for k in envs}
    for _ in range(args.rounds):
        for k, env in envs.items():
            res[k].append(episode(torch, env.stepper, T, 7))
    on = envs["on"]
    out = dict(workload="c4", envs=args.envs, episode_length=T, rounds=args.rounds, gpu=gpu, arms={},
               metrics_tensor_ms=call_ms(torch, lambda o=None: on.metrics_tensor(out=o)),
               previous_episode_metrics_tensor_ms=call_ms(torch, lambda o=None: on.previous_episode_metrics_tensor(out=o)))
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
    for k, arm in out["arms"].items():
        print("%-4s" % k, "  ".join("%s %.4f (%.4f-%.4f) %+.1f%%" % (f, arm[f]["median"], *arm[f]["range"],
                                                                     100.0 * (arm[f]["median"] / off[f]["median"] - 1.0))
                                    for f in fields))
    print("metrics_tensor() ms:", out["metrics_tensor_ms"], "| card (name, power limit, max SM clock):", gpu)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
