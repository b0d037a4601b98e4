"""Times env checkpoints on cuda:0: `env.state_dict()` + `torch.save` (save), and `torch.load` + `load_state_dict()` into
a second env of the same configuration made beforehand (load), with the host clock around each, ending in a device
synchronise.  The checkpoint goes to a temporary directory (page cache, not a durable write).  Prints the card's name and
power limit, then per workload the checkpoint's bytes and the median and range of each time over the rounds.

    python tools/time_checkpoint.py [--workloads c2,c3,c5,c4] [--rounds 5] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai_economist_b200 import foundation  # noqa: E402
from ai_economist_b200.workloads import product_kwargs  # noqa: E402

WORKLOADS = {"c2": ("c1_tutorial", 8192, {}), "c3": ("c3_paper_tax", 8192, {}),
             "c5": ("c5_full", 2048, dict(device_reset="snapshot")), "c4": ("covid", 4096, {})}


def make(cfg, E, extra, seed):
    if cfg == "covid":
        from ai_economist_b200.workloads import COVID_KWARGS, covid_reference_config
        kw = covid_reference_config(dict(COVID_KWARGS))
        return foundation.make_env_instance(kw.pop("scenario_name"), n_envs=E, device="cuda:0", **kw)
    name, kw = product_kwargs(cfg)
    return foundation.make_env_instance(name, n_envs=E, device="cuda:0", seed=seed, **extra, **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3,c5,c4")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_checkpoint.py measures on a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    results = {"card": q, "workloads": {}}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "env.pt")
        for wl in a.workloads.split(","):
            cfg, E, extra = WORKLOADS[wl]
            src, dst = make(cfg, E, extra, 1), make(cfg, E, extra, 2)
            src.reset()
            for _ in range(5):
                src.stepper.sample_random_actions(seed=3)
                src.step(src.action_buffers)
            torch.cuda.synchronize()
            save, load = [], []
            for _ in range(a.rounds):
                t0 = time.perf_counter()
                torch.save(src.state_dict(), path)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                dst.load_state_dict(torch.load(path, weights_only=False))
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                save.append(1e3 * (t1 - t0))
                load.append(1e3 * (t2 - t1))
            nbytes = os.path.getsize(path)
            med = lambda v: sorted(v)[len(v) // 2]
            r = dict(envs=E, bytes=nbytes, save_ms=med(save), save_ms_range=[min(save), max(save)], load_ms=med(load),
                     load_ms_range=[min(load), max(load)])
            results["workloads"][wl] = r
            print("%s (%d replicas): %.1f MB; state_dict + torch.save %.1f ms [%.1f, %.1f]; torch.load + load_state_dict "
                  "%.1f ms [%.1f, %.1f]" % (wl, E, nbytes / 1e6, r["save_ms"], *r["save_ms_range"], r["load_ms"],
                                            *r["load_ms_range"]), flush=True)
            del src, dst
            torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
