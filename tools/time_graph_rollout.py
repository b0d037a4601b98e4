"""Times a captured rollout (env.capture_rollout) against the eager bound loop it records, on cuda:0.

Arms, alternated over rounds on one env, with tools/time_rollout.py's policy heads (one linear layer each):
  eager  restart_rollout(), then T x (sample_actions over the heads' logits, step) into the bound rollout;
  graph  restart_rollout(), then one replay() of those T iterations recorded once by capture_rollout.
Each arm's time is the host clock over `--reps` rollouts ending in a device synchronise.  Workloads: c2 / c3 (8 192
replicas), c5 (2 048), c4 (COVID-19, 4 096), and c2 / c4 at 512 replicas, where launch overhead weighs most.

A separate run per workload (--enqueue) times the eager loop's host enqueue per step (host clock over T steps with no
synchronise, the queue drained before) against its device time per step (CUDA events around the same T steps): an
enqueue time close to the device time means the loop is bound by the host.  Prints the card's name and power limit,
then per workload the median and range of ms per step of each arm.

    python tools/time_graph_rollout.py [--workloads c2,c3,c5,c4,c2_512,c4_512] [--T 16] [--rounds 5] [--reps 4]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_rollout import CovidNets, Nets, make, obs_tensors  # noqa: E402

WORKLOADS = {"c2": ("c1_tutorial", 8192), "c3": ("c3_paper_tax", 8192), "c5": ("c5_full", 2048), "c4": ("covid", 4096),
             "c2_512": ("c1_tutorial", 512), "c4_512": ("covid", 512)}
SEED = 7


def eager(env, nets, T):
    env.restart_rollout()
    for t in range(T):
        env.sample_actions(*nets.logits(obs_tensors(env)), seed=SEED)
        env.step(env.action_buffers)


def replay(env, graph):
    env.restart_rollout()
    graph.replay()


def timed(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def enqueue_vs_device(env, nets, T, reps):
    """Host enqueue ms / step (no synchronise inside) and device ms / step (events) of the eager loop, medians."""
    host, dev = [], []
    for _ in range(reps):
        env.restart_rollout()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for t in range(T):
            env.sample_actions(*nets.logits(obs_tensors(env)), seed=SEED)
            env.step(env.action_buffers)
        e1.record()
        host.append((time.perf_counter() - t0) * 1e3 / T)
        torch.cuda.synchronize()
        dev.append(e0.elapsed_time(e1) / T)
    return statistics.median(host), statistics.median(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3,c5,c4,c2_512,c4_512")
    ap.add_argument("--T", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--enqueue", action="store_true", help="time host enqueue against device time instead")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card:", q)
    for wl in a.workloads.split(","):
        cfg, E = WORKLOADS[wl]
        env = make(cfg, E)
        nets = CovidNets(env) if cfg == "covid" else Nets(env)
        env.bind_rollout(a.T, final_obs=True)
        env.reset()
        for _ in range(a.T):   # warm-up: the slots' shapes, cuBLAS's algorithms
            env.sample_actions(*nets.logits(obs_tensors(env)), seed=SEED)
            env.step(env.action_buffers)
        if a.enqueue:
            h, d = enqueue_vs_device(env, nets, a.T, a.rounds * a.reps)
            print("%-7s E=%5d T=%d eager loop: host enqueue %.4f ms/step, device %.4f ms/step (%s)"
                  % (wl, E, a.T, h, d, "host-bound" if h >= 0.9 * d else "device-bound"))
        else:
            env.restart_rollout()
            graph = env.capture_rollout(lambda t, obs: env.sample_actions(*nets.logits(obs), seed=SEED))
            graph.replay()   # the capture leaves the cursor at 0
            eager(env, nets, a.T)
            ms = {"eager": [], "graph": []}
            for r in range(a.rounds):
                arms = [("eager", lambda: eager(env, nets, a.T)), ("graph", lambda: replay(env, graph))]
                for name, fn in (arms if r % 2 == 0 else arms[::-1]):
                    ms[name].append(timed(fn, a.reps) / (a.reps * a.T))
            line = "%-7s E=%5d T=%d" % (wl, E, a.T)
            for name in ("eager", "graph"):
                v = ms[name]
                line += "  %s %.4f ms/step [%.4f, %.4f]" % (name, statistics.median(v), min(v), max(v))
            print(line + "  ratio %.3f" % (statistics.median(ms["graph"]) / statistics.median(ms["eager"])))
        del env
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
