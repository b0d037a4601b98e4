"""Cost of reading episode metrics on the GPU: the batched path (env.metrics_tensor / previous_episode_metrics_tensor, one
kernel launch) against the per-replica path (env.metrics_of / previous_episode_metrics_of: a device synchronise, a record
copy and a Python dict per replica).

For each workload (bench.py's c2 / c3 at 8192 replicas, c5 at 2048 with the snapshot device reset), with episode phases staggered as in bench.py
(replica e starts at t = e*T/E, then one untimed episode of steps under the fused random policy):
  (a) the batched call's device time (CUDA events over many calls) and its bytes: whole records read (an upper bound on
      what the kernel touches) + E x K x 8 written;
  (b) host-clock time of the per-replica path for the replicas that finished in one step, and for all replicas;
  (c) ms per step of a stepping loop that logs the finished episodes' metrics every step, per-replica path against
      batched path, alternated in one session.
Prints one JSON object (and writes it to --out).  GPU only: there is no CPU fallback.

usage: python tools/time_batched_metrics.py [--workloads c2,c3,c5] [--calls 200] [--loop-steps 200] [--rounds 2] [--out F]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from ai_economist_b200 import foundation  # noqa: E402
from ai_economist_b200.workloads import product_kwargs  # noqa: E402

# (configuration, replicas, device reset) as bench.py runs them
WORKLOADS = {"c2": ("c1_tutorial", 8192, None), "c3": ("c3_paper_tax", 8192, None), "c5": ("c5_full", 2048, "snapshot")}


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["nvidia_smi"] = q
    except Exception as ex:  # noqa: BLE001
        out["nvidia_smi"] = "unavailable: %r" % ex
    return out


def make_env(workload):
    cfg, E, reset = WORKLOADS[workload]
    name, kw = product_kwargs(cfg)
    if reset:
        kw["device_reset"] = reset
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", seeds=list(range(1000, 1000 + E)),
                                       auto_reset=True, **kw)
    env.reset()
    st, T = env.stepper, env.episode_length
    st.state_view("t").copy_((torch.arange(E, device="cuda:0", dtype=torch.int64) * T // E).to(torch.int32))
    st.set_fused_policy(1234)
    for _ in range(T):
        st.step()
    torch.cuda.synchronize()
    return env


def batched_call(env, calls):
    st, E = env.stepper, env.n_envs
    K = len(env.metric_keys)
    out = torch.empty((E, K), dtype=torch.float64, device="cuda:0")
    res = {}
    for final in (False, True):
        for _ in range(10):
            st.episode_metrics(final=final, out=out)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = st.launch_count()
        a.record()
        for _ in range(calls):
            st.episode_metrics(final=final, out=out)
        b.record()
        b.synchronize()
        assert st.launch_count() - n0 == calls
        ms = a.elapsed_time(b) / calls
        res["previous_episode" if final else "current"] = dict(device_ms_per_call=ms)
    rec = int(st.dims.state_bytes)
    res.update(K=K, record_bytes=rec, bytes_read_records=E * rec, bytes_written=E * K * 8,
               gb_per_s_upper=(E * rec + E * K * 8) / (res["current"]["device_ms_per_call"] * 1e-3) / 1e9)
    return res


def per_replica(env, max_all_seconds):
    st = env.stepper
    st.step()
    torch.cuda.synchronize()
    done = torch.nonzero(st.buf["done"]).flatten().tolist()
    t0 = time.perf_counter()
    for e in done:
        env.previous_episode_metrics_of(e)
    t_done = time.perf_counter() - t0
    t0, n = time.perf_counter(), 0
    for e in range(env.n_envs):
        env.metrics_of(e)
        n += 1
        if time.perf_counter() - t0 > max_all_seconds:
            break
    t_all = time.perf_counter() - t0
    return dict(finished_in_step=len(done), finished_ms=1e3 * t_done,
                finished_ms_per_replica=1e3 * t_done / max(1, len(done)),
                all_replicas_measured=n, all_ms_measured=1e3 * t_all, all_ms_per_replica=1e3 * t_all / n,
                all_ms_extrapolated=1e3 * t_all / n * env.n_envs)


def logging_loop(env, steps, rounds):
    """ms per step of stepping + logging the metrics of the episodes that ended in each step."""
    st = env.stepper
    K = len(env.metric_keys)
    buf = torch.empty((env.n_envs, K), dtype=torch.float64, device="cuda:0")
    acc = torch.zeros(K, dtype=torch.float64, device="cuda:0")
    cnt = torch.zeros((), dtype=torch.float64, device="cuda:0")

    def per_replica_step():
        st.step()
        for e in torch.nonzero(st.buf["done"]).flatten().tolist():   # synchronises on the done flags
            env.previous_episode_metrics_of(e)

    def batched_step():
        st.step()
        m = env.previous_episode_metrics_tensor(out=buf)
        d = st.buf["done"].bool()
        acc.add_(torch.where(d[:, None], m, torch.zeros((), dtype=m.dtype, device=m.device)).sum(0))  # no sync
        cnt.add_(d.sum())

    def plain_step():
        st.step()

    arms = {"per_replica": per_replica_step, "batched": batched_step, "no_logging": plain_step}
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            for _ in range(10):
                fn()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                fn()
            torch.cuda.synchronize()
            res[name].append(1e3 * (time.perf_counter() - t0) / steps)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3,c5")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--loop-steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--max-all-seconds", type=float, default=30.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_batched_metrics.py needs a CUDA device")
    result = {"card": card(), "workloads": {}}
    for w in args.workloads.split(","):
        env = make_env(w)
        r = dict(n_envs=env.n_envs, n_agents=env.n_agents)
        r["batched"] = batched_call(env, args.calls)
        r["per_replica"] = per_replica(env, args.max_all_seconds)
        r["logging_loop_ms_per_step"] = logging_loop(env, args.loop_steps, args.rounds)
        result["workloads"][w] = r
        print(json.dumps({w: r}), flush=True)
        env.stepper.close()
        del env
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
