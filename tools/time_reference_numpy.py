"""Times the UNMODIFIED reference's own NumPy `env.step()` (imported from a reference checkout, oracle/ref_harness.py) on
the BASELINE configurations, one process per allowed core, and prints the rates as JSON - the number the north star asks
to be reported beside the GPU rate.  The reference is pure Python and is not part of this repository, so it is timed
wherever a checkout exists, with the host's core count stated.

    python tools/time_reference_numpy.py [--steps 300]
"""
import argparse
import json
import multiprocessing as mp
import os
import platform
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def worker(args):
    cfg_name, steps, seed, cpu = args
    try:
        os.sched_setaffinity(0, {cpu})
    except Exception:
        pass
    from oracle import ref_harness as rh
    from oracle.configs import CONFIGS
    f = rh.load_reference_foundation()
    kw = dict(CONFIGS[cfg_name])
    np.random.seed(seed)
    env = f.make_env_instance(**kw)
    obs = env.reset()
    rng = np.random.RandomState(seed)
    total, n = 0.0, 0
    for t in range(steps + 5):
        acts = rh.sample_actions(env, obs, rng)[0]  # sampling excluded from the timed region
        t0 = time.perf_counter()
        obs, rew, done, info = env.step(acts)
        dt = time.perf_counter() - t0
        if t >= 5:
            total += dt
            n += 1
        if done["__all__"]:
            obs = env.reset()
    return n / total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    a = ap.parse_args()
    cpus = sorted(os.sched_getaffinity(0))
    out = {"what": "the reference's own NumPy BaseEnvironment.step(), unmodified, imported from /root/reference; one "
                   "process per allowed core, each pinned, stepping its own env with uniformly random unmasked actions; "
                   "env.step only (action sampling excluded)",
           "where": "build container (the reference cannot travel to the GPU box)", "host": platform.processor() or platform.machine(),
           "cores": len(cpus), "numpy": np.__version__, "steps_per_process": a.steps, "configs": {}}
    agents = {"c1_tutorial": 4, "c3_paper_tax": 10, "c5_full": 64}
    for cfg, key in (("c1_tutorial", "c2"), ("c3_paper_tax", "c3"), ("c5_full", "c5")):
        steps = a.steps if key != "c5" else max(20, a.steps // 10)
        with mp.Pool(len(cpus)) as pool:
            rates = pool.map(worker, [(cfg, steps, 100 + i, c) for i, c in enumerate(cpus)])
        per_core = float(np.mean(rates))
        out["configs"][key] = {"env_steps_per_s_per_core": per_core, "env_steps_per_s_all_cores": float(np.sum(rates)),
                               "agent_env_steps_per_s_all_cores": float(np.sum(rates)) * agents[cfg], "n_agents": agents[cfg]}
        print(key, out["configs"][key], flush=True)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
