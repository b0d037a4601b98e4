"""Time an explicit env.reset() at the benchmark's sizes: the host path (the scenario's host_reset per replica, packed
and uploaded by load_host_state) against the device path (aie_reset_envs: one launch re-draws every replica, one launch
writes the observations), for the first reset and for a later one.  Default (reference-exact) reset mode.

python tools/time_reset.py [--configs c2,c3,c5] [--repeat 10] [--host-envs N]

Host path and first device reset: host clock around the call, ending in torch.cuda.synchronize().  Later device
reset: the same, averaged over --repeat calls, plus the device time of the two launches alone (CUDA events around a
stepper.reset_envs() call).  --host-envs N times the host path on the first N replicas only and scales it to the full
batch (the output says so).  Prints the card name and power limit of the same run, then one JSON line per config."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {"c2": ("c1_tutorial", 8192), "c3": ("c3_paper_tax", 8192), "c5": ("c5_full", 2048)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make(cfg_name, E):
    from ai_economist_b200 import foundation, workloads
    from oracle.configs import CONFIGS as TABLE
    name, kw = workloads.product_kwargs(cfg_name, TABLE)
    env = foundation.make_env_instance(name, n_envs=E, device="cuda:0", auto_reset=False, **kw)
    env.seed(1000)
    assert env.spec["reset_mode"] == 1, "the device path needs a reference-exact reset"
    return env


def time_config(key, repeat, host_envs):
    import torch
    cfg_name, E = CONFIGS[key]
    res = {"config": key, "envs": E}

    warm = make(cfg_name, 2)   # loads the kernels: the first timed reset measures the reset, not module loading
    warm.reset()
    del warm
    # device path: first reset (template + streams uploaded), then later resets from the records
    env = make(cfg_name, E)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    env.reset()
    torch.cuda.synchronize()
    res["device_first_ms"] = 1e3 * (time.perf_counter() - t0)
    env.reset()   # warm-up of the later path
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(repeat):
        env.reset()
    torch.cuda.synchronize()
    res["device_later_ms"] = 1e3 * (time.perf_counter() - t0) / repeat
    st = env.stepper
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(repeat):
        st.reset_envs()
    ev1.record()
    torch.cuda.synchronize()
    res["device_later_kernels_ms"] = ev0.elapsed_time(ev1) / repeat
    n0 = st.launch_count()
    env.reset()
    res["device_later_launches"] = st.launch_count() - n0
    del env, st
    torch.cuda.empty_cache()

    # host path: host_reset per replica + pack + upload (what reset() ran before), on the first n replicas
    env = make(cfg_name, E)
    n = E if not host_envs else min(E, host_envs)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    env.n_envs = n   # host_reset_arrays() walks replicas 0 .. n_envs - 1
    try:
        arrays = env.host_reset_arrays()
    finally:
        env.n_envs = E
    env.load_host_state(arrays)
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t0)
    res["host_ms"] = ms * E / n
    res["host_measured_envs"] = n
    if n != E:
        res["host_note"] = "measured on %d replicas and scaled to %d: not measured at full size" % (n, E)
    del env
    torch.cuda.empty_cache()
    res["speedup_first"] = res["host_ms"] / res["device_first_ms"]
    res["speedup_later"] = res["host_ms"] / res["device_later_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3,c5")
    ap.add_argument("--repeat", type=int, default=10)
    ap.add_argument("--host-envs", type=int, default=0, help="time the host path on this many replicas (0: all)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("time_reset.py measures on a CUDA device; none is visible")
    print("card:", card(), flush=True)
    for key in args.configs.split(","):
        print(json.dumps(time_config(key, args.repeat, args.host_envs)), flush=True)


if __name__ == "__main__":
    main()
