"""TEST INFRASTRUCTURE: record the reference's COVID-19 episode metrics (CovidAndEconomySimulation.scenario_metrics(),
covid19_env.py:1613-1687) along the action sequences of the recorded COVID-19 traces, from the UNMODIFIED reference
(build container only), into tests/golden/covid_metrics/<trace>.npz.  Data only: meta_json (the trace, its kwargs,
episode_length, n_steps), keys (the metrics keys in the reference's dict order), and per point n (steps taken since the
first reset), end (taken at an episode end) and values (float64, in key order).

The three single-episode traces (tests/golden_covid/) are recorded at several t and after their last step (the episode
end).  The six variant traces (tests/golden/covid_variants/) run across episode ends with a reset at each, as they were
recorded: at each end the metrics are taken before env.reset() (end set), and mid-episode points of every episode
after a reset show what the reference returns then (global_state is rebuilt by the reset, so its rows after t are zero).
Usage: python oracle/gen_golden_covid_metrics.py
"""
import contextlib
import glob
import io
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness as rh  # noqa: E402
from oracle.gen_golden_covid import reference_config  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "covid_metrics")
TRACES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden_covid", "*.npz"))) + \
    sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "covid_variants", "*.npz")))


def points_of(T, n_steps):
    """Step counts n at which mid-episode metrics are taken: t = 1, a third and two thirds of the episode, T - 1."""
    pts = set()
    for start in range(0, n_steps, T):
        for t in (1, T // 3, (2 * T) // 3, T - 1):
            if 1 <= t < T and start + t <= n_steps:
                pts.add(start + t)
    return pts


def as_float(m):
    return [float(np.asarray(v).reshape(-1)[0]) for v in m.values()]


def record(path):
    d = np.load(path)
    meta = json.loads(str(d["meta_json"]))
    kw = meta["kwargs"]
    T, n_steps = int(kw["episode_length"]), int(meta["n_steps"])
    f = rh.load_reference_foundation()
    with contextlib.redirect_stdout(io.StringIO()):
        env = f.make_env_instance(**reference_config(kw))
        env.reset()
    pts = points_of(T, n_steps)
    out, keys = [], None
    for n in range(1, n_steps + 1):
        actions = {str(i): int(d["act_a"][n - 1][i]) for i in range(51)}
        actions["p"] = int(d["act_p"][n - 1])
        _, _, done, _ = env.step(actions)
        if done["__all__"]:
            m = env.scenario_metrics()
            keys = list(m)
            out.append(dict(n=n, end=True, values=as_float(m)))
            if meta.get("reset_at_done"):
                with contextlib.redirect_stdout(io.StringIO()):
                    env.reset()
        elif n in pts:
            m = env.scenario_metrics()
            keys = list(m)
            out.append(dict(n=n, end=False, values=as_float(m)))
    return dict(trace=os.path.relpath(path, ROOT), kwargs=kw, episode_length=T, n_steps=n_steps,
                reset_at_done=bool(meta.get("reset_at_done")), keys=keys, points=out)


def main():
    os.makedirs(OUT, exist_ok=True)
    for path in TRACES:
        rec = record(path)
        pts, keys = rec.pop("points"), rec.pop("keys")
        dst = os.path.join(OUT, os.path.splitext(os.path.basename(path))[0] + ".npz")
        np.savez_compressed(dst, meta_json=np.array(json.dumps(rec)), keys=np.array(keys),
                            n=np.array([q["n"] for q in pts], np.int32), end=np.array([q["end"] for q in pts], bool),
                            values=np.array([q["values"] for q in pts], np.float64))
        print(dst, len(pts), "points", "%.1f KB" % (os.path.getsize(dst) / 1024))


if __name__ == "__main__":
    main()
