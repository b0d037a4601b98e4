"""TEST INFRASTRUCTURE: generate tests/golden/*.npz from the UNMODIFIED reference.

Runs in the build container only (needs /root/reference).  Each fixture holds
  * spec_json    — flat config dict (oracle/ref_harness.spec_from_reference_env) + the reference kwargs
  * init_*       — post-reset host snapshot (maps, locs, skills, numpy MT19937 state)
  * act_a/act_p  — the action trace (sampled from a separate RandomState over unmasked actions)
  * per-step compact state (exact ints + float64 coin/labor/...), rewards,
    CRC32 of every exact-valued observation array, and the full float observations every
    `full_every` steps (and at the last step).
Usage: python oracle/gen_golden.py
"""
import json
import os
import sys
import zlib

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402
from oracle.configs import CONFIGS  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

# (config, seed, steps, full_every)
PLAN = [
    ("c1_tutorial", 1001, 1000, 25),
    ("c1_tutorial", 1002, 300, 25),
    ("c3_paper_tax", 1001, 450, 50),
    ("c3_short_period", 1001, 200, 10),
    ("tax_us_federal", 1001, 120, 10),
    ("ref_unit_test", 1001, 100, 10),
    ("c5_small", 1001, 150, 25),
    ("c5_full", 1001, 60, 20),
    ("wealth_redistribution", 1001, 300, 25),
    ("multi_zone", 1001, 120, 20),
    ("quadrant", 1001, 120, 20),
    ("split_layout", 1001, 120, 20),
    ("tax_single_planner", 1001, 150, 10),
    ("uniform_halfwidth", 1001, 150, 25),
    ("full_obs_tax", 1001, 100, 20),
    # multi-episode traces (env.reset() between episodes, the global numpy stream continues): device-side reset
    ("c1_reset", 1001, 80, 10),
    ("c3_reset", 1001, 95, 10),
    ("saez_reset", 1001, 790, 50),
    ("saez_annealed_reset", 1001, 790, 50),
    ("lognormal_reset", 1001, 95, 10),
    ("split_reset", 1001, 90, 10),
    ("us_federal_annealed_reset", 1001, 90, 5),
    ("uniform_reset", 1001, 100, 10),
    ("quadrant_reset", 1001, 95, 7),
    ("multi_zone_reset", 1001, 90, 8),
]

# tests/test_oracle_vs_reference.py: other seeds and lengths, full observations at every step
PLAN_LIVE = [
    ("c1_tutorial", 31, 150, 1),
    ("c3_short_period", 32, 120, 1),
    ("c5_small", 33, 40, 1),
    ("ref_unit_test", 34, 60, 1),
]

EXACT_OBS = ["a_map", "a_idx", "a_mask", "p_map", "p_idx", "p_mask"]
FLOAT_OBS = ["a_flat", "p_flat", "p_agents", "time"]
STEP_STATE = ["loc", "inv", "esc", "coin", "esc_coin", "labor", "n_orders", "tax_pos", "rate_idx",
              "last_coin", "last_income", "last_marg", "mt_pos"]


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a).tobytes()) & 0xFFFFFFFF


def generate(cfg_name, seed, steps, full_every, out_dir=None):
    f = rh.load_reference_foundation()
    cfg = dict(CONFIGS[cfg_name])
    env = f.make_env_instance(**cfg)
    env.seed(seed)
    obs = env.reset()
    spec = rh.spec_from_reference_env(env)
    init = rh.state_from_reference_env(env)
    arng = np.random.RandomState(seed + 7919)
    rec = {k: [] for k in STEP_STATE + ["rew", "done", "cell_crc", "owner_crc", "book_crc", "hist_crc",
                                          "price_hist_sum", "mt_key_crc"]}
    rec.update({k + "_crc": [] for k in EXACT_OBS})
    full = {k: [] for k in FLOAT_OBS + EXACT_OBS}
    full_steps = []
    acts_a, acts_p = [], []

    def snapshot(t, obs, rew, done, force_full=False):
        ro = rh.obs_arrays_from_reference(env, obs, rew, done)
        rs = rh.state_arrays_from_reference(env)
        for k in STEP_STATE:
            if k in rs:
                rec[k].append(np.array(rs[k]))
        rec["rew"].append(ro.get("rew", np.zeros(env.n_agents + 1)))
        rec["done"].append(int(ro["done"][0]) if "done" in ro else 0)
        rec["cell_crc"].append(crc(rs["cell"]))
        rec["owner_crc"].append(crc(rs["owner"]))
        rec["mt_key_crc"].append(crc(rs["mt_key"]))
        if "book" in rs:
            rec["book_crc"].append(crc(np.concatenate([rs["book"][(c, s)].ravel() for c in (0, 1) for s in (0, 1)]
                                                      + [np.zeros(1, np.int32)])))
            rec["hist_crc"].append(crc(np.concatenate([rs["bid_hist"].ravel(), rs["ask_hist"].ravel()])))
            rec["price_hist_sum"].append(float(rs["price_hist"].sum()))
        for k in EXACT_OBS:
            if k in ro:
                rec[k + "_crc"].append(crc(ro[k]))
        if force_full or t % full_every == 0:
            full_steps.append(t)
            for k in FLOAT_OBS + EXACT_OBS:
                if k in ro:
                    full[k].append(ro[k])

    snapshot(0, obs, None, None, force_full=True)
    for t in range(1, steps + 1):
        actions, a_act, p_act = rh.sample_actions(env, obs, arng)
        obs, rew, done, _ = env.step(actions)
        if done["__all__"] and t < steps:
            obs = env.reset()   # reference semantics: a fresh episode drawn from the same (continuing) global stream
        acts_a.append(a_act)
        acts_p.append(p_act)
        snapshot(t, obs, rew, done, force_full=(t == steps))

    out = {"spec_json": np.array(json.dumps(dict(spec=spec, reference_kwargs=cfg, seed=seed, n_steps=steps)))}
    for k, v in init.items():
        out["init_" + k] = np.asarray(v)
    out["act_a"] = np.stack(acts_a).astype(np.int8)
    out["act_p"] = np.stack(acts_p).astype(np.int16)   # single-action planner indices exceed int8
    for k, v in rec.items():
        if v:
            out["step_" + k] = np.stack([np.asarray(x) for x in v])
    out["full_steps"] = np.array(full_steps, np.int32)
    for k, v in full.items():
        if v:
            arr = np.stack(v)
            if k in ("a_map", "p_map"):
                arr = arr.astype(np.uint8)  # 0/1-valued float32 planes: stored as u8, compared after cast
            out["full_" + k] = arr
    if out_dir is None:
        out_dir = OUT + "_reset" if cfg_name.endswith("_reset") else OUT   # multi-episode traces live apart
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "%s_seed%d.npz" % (cfg_name, seed))
    np.savez_compressed(path, **out)
    print("%s: %d steps, %.1f KB" % (path, steps, os.path.getsize(path) / 1024))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    only = set(sys.argv[1:])   # optional: config names to (re)generate
    for item in PLAN:
        if not only or item[0] in only:
            generate(*item)
    for item in PLAN_LIVE:
        if not only or item[0] in only:
            generate(*item, out_dir=os.path.join(OUT, "live"))
