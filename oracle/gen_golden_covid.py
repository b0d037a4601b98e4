"""TEST INFRASTRUCTURE: record a COVID-19 golden trace from the UNMODIFIED reference (build container only) and,
with --check, step oracle/covid_oracle.py beside it.  Config = tests/run_covid19_cpu_gpu_consistency_checks.py:44-81.
Usage: python oracle/gen_golden_covid.py [--check] [--steps N]
       python oracle/gen_golden_covid.py --variant NAME [--check]     (one of VARIANTS, into tests/golden/covid_variants/)

A variant trace runs across episode ends: the step that returns `done` records that step's rewards and `done`, then
env.reset() and records the reset observation as that step's observation (what the product's auto-reset returns), and
the trace goes on into the next episode: two full episodes and VARIANT_EXTRA_STEPS steps of the third.
"""
import argparse
import contextlib
import io
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden_covid")
VARIANT_OUT = os.path.join(os.path.dirname(OUT), "golden", "covid_variants")

from ai_economist_b200.workloads import COVID_KWARGS, covid_reference_config  # noqa: E402

# Parameter variants of the COVID workload: name -> (action seed, kwargs over COVID_KWARGS).  Each reaches device code
# the default parameters do not:
#   eta3_cooldown1_levels1      x ** -2 through the general powf; a 2-entry planner segment; vaccine deliveries that began
#                               before the start date (every 7th day from day 7); change lists overflowing (cooldown 1)
#   eta05_cooldown7_interval1   x ** 0.5 (the sqrt path); a planner mask open at every step
#   eta15_levels40_health       x ** -0.5 through the general powf; a 41-entry planner segment (longer than a warp);
#                               other health weights
#   cooldown1_len60             the defaults with 1-day cooldowns: auto-reset of overflowed change lists
#   early_start_daily_vaccines  the initial history window padded before the data begins; daily deliveries from day 10
#   late_start_window_drops     the last start date with complete data: the real-world changes of the initial window reach its
#                               oldest index and leave it (from step 121), so change-list entries drop off the front
VARIANTS = {
    "eta3_cooldown1_levels1": (21, dict(
        episode_length=50, economic_reward_crra_eta=3.0, action_cooldown_period=1, subsidy_interval=30,
        num_subsidy_levels=1, start_date="2020-10-15", vaccine_delivery_start_date="2020-07-01", delivery_interval=7,
        daily_vaccines_per_million_people=10000)),
    "eta05_cooldown7_interval1": (22, dict(
        episode_length=40, economic_reward_crra_eta=0.5, action_cooldown_period=7, subsidy_interval=1,
        num_subsidy_levels=5, start_date="2020-06-01")),
    "eta15_levels40_health": (23, dict(
        episode_length=70, economic_reward_crra_eta=1.5, action_cooldown_period=28, num_subsidy_levels=40,
        subsidy_interval=30, health_priority_scaling_agents=1.0, health_priority_scaling_planner=2.0)),
    "cooldown1_len60": (24, dict(episode_length=60, action_cooldown_period=1)),
    "early_start_daily_vaccines": (25, dict(
        episode_length=45, economic_reward_crra_eta=2, start_date="2020-03-22", daily_vaccines_per_million_people=10000,
        delivery_interval=1, vaccine_delivery_start_date="2020-04-01", subsidy_interval=90)),
    "late_start_window_drops": (26, dict(episode_length=130, start_date="2021-04-30", subsidy_interval=45)),
}
VARIANT_EXTRA_STEPS = 5


def variant_kwargs(name):
    """(full kwargs, action seed) of a named variant"""
    seed, over = VARIANTS[name]
    return dict(COVID_KWARGS, **over), seed


def variant_path(name):
    return os.path.join(VARIANT_OUT, "%s.npz" % name)


def reference_config(kw):
    return covid_reference_config(kw)


def ref_arrays(env, obs, rew=None, done=None):
    a, p = obs["a"], obs["p"]
    out = dict(
        agent_state=np.asarray(a["world-agent_state"], np.float32),
        postsubsidy=np.asarray(a["world-agent_postsubsidy_productivity"], np.float32),
        lagged=np.asarray(a["world-lagged_stringency_level"], np.float32),
        policy_ind=np.asarray(a["ControlUSStateOpenCloseStatus-agent_policy_indicators"], np.float32),
        scalars=np.array([np.asarray(p["time"]).ravel()[0], p["FederalGovernmentSubsidy-t_until_next_subsidy"],
                          p["FederalGovernmentSubsidy-current_subsidy_level"],
                          p["VaccinationCampaign-t_until_next_vaccines"]], np.float32),
        mask_a=np.asarray(a["action_mask"], np.float32), mask_p=np.asarray(p["action_mask"], np.float32))
    # planner copies / broadcast vectors must agree with the agent-side fields
    assert np.array_equal(np.asarray(p["world-agent_state"]), np.asarray(a["world-agent_state"]))
    assert np.allclose(np.asarray(a["time"]), out["scalars"][0])
    assert np.allclose(np.asarray(a["FederalGovernmentSubsidy-t_until_next_subsidy"]), out["scalars"][1])
    assert np.array_equal(np.asarray(a["world-agent_index"]), np.eye(51, dtype=np.int32))
    if rew is not None:
        out["rew_a"] = np.asarray(rew["a"], np.float32)
        out["rew_p"] = np.float64(rew["p"])
        out["done"] = np.int32(done["__all__"])
    gs = env.world.global_state
    t = env.world.timestep
    out["st_susceptible"], out["st_infected"], out["st_deaths"] = gs["Susceptible"][t], gs["Infected"][t], gs["Deaths"][t]
    out["st_unemployed"], out["st_stringency"], out["st_subsidy"] = gs["Unemployed"][t], gs["Stringency Level"][t], gs["Subsidy"][t]
    return {k: np.array(v) for k, v in out.items()}


def sample(obs, rng):
    ma = np.asarray(obs["a"]["action_mask"])  # [11, 51]
    mp = np.asarray(obs["p"]["action_mask"])  # [21]
    act_a = np.array([rng.choice(ma.shape[0], p=ma[:, i] / ma[:, i].sum()) for i in range(ma.shape[1])], np.int32)
    act_p = np.int32(rng.choice(len(mp), p=mp / mp.sum()))
    return act_a, act_p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--steps", type=int, default=540)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--cooldown", type=int, default=None, help="action_cooldown_period of the variant (default: the workload's 28)")
    ap.add_argument("--episode-length", type=int, default=None)
    ap.add_argument("--name", default=None, help="file name stem (default covid_seed<seed>)")
    ap.add_argument("--variant", default=None, choices=sorted(VARIANTS),
                    help="record the named variant across two episode ends (ignores --steps, --seed, --cooldown, --episode-length)")
    args = ap.parse_args()
    kwargs = dict(COVID_KWARGS)
    multi_episode = args.variant is not None
    if multi_episode:
        kwargs, args.seed = variant_kwargs(args.variant)
        args.steps = 2 * kwargs["episode_length"] + VARIANT_EXTRA_STEPS
    if args.cooldown is not None and not multi_episode:
        kwargs["action_cooldown_period"] = args.cooldown
    if args.episode_length is not None and not multi_episode:
        kwargs["episode_length"] = args.episode_length
        args.steps = min(args.steps, args.episode_length)
    f = rh.load_reference_foundation()
    with contextlib.redirect_stdout(io.StringIO()):
        env = f.make_env_instance(**reference_config(kwargs))
        obs = env.reset()
    orc = None
    if args.check:
        from ai_economist_b200.foundation.covid19 import build_covid_params
        from oracle.covid_oracle import CovidOracleEnv
        orc = CovidOracleEnv(build_covid_params(**kwargs), auto_reset=multi_episode)
    rng = np.random.RandomState(args.seed)
    rec = {k: [v] for k, v in ref_arrays(env, obs).items()}
    acts_a, acts_p = [], []

    def check(t, ra):
        oo = orc.obs()
        for k in ["agent_state", "postsubsidy", "lagged", "policy_ind", "scalars", "mask_a", "mask_p"] + \
                 (["rew_a", "rew_p", "done"] if t else []):
            if not np.allclose(ra[k], oo[k], rtol=1e-6, atol=1e-9):
                bad = np.argwhere(~np.isclose(ra[k], oo[k], rtol=1e-6, atol=1e-9))[:3]
                raise SystemExit("step %d: %s differs at %s ref=%s orc=%s" % (t, k, bad.tolist(), np.asarray(ra[k]).ravel()[:3], np.asarray(oo[k]).ravel()[:3]))
        exact = all(np.array_equal(ra[k], oo[k]) for k in ["agent_state", "postsubsidy", "mask_a"])
        return exact

    n_exact = 0
    if orc:
        n_exact += check(0, {k: v[0] for k, v in rec.items()})
    for t in range(1, args.steps + 1):
        act_a, act_p = sample(obs, rng)
        actions = {str(i): int(act_a[i]) for i in range(51)}
        actions["p"] = int(act_p)
        obs, rew, done, _ = env.step(actions)
        acts_a.append(act_a); acts_p.append(act_p)
        if multi_episode and done["__all__"]:
            with contextlib.redirect_stdout(io.StringIO()):
                obs = env.reset()
        ra = ref_arrays(env, obs, rew, done)
        for k, v in ra.items():
            rec.setdefault(k, []).append(v)
        if orc:
            orc.step(act_a, act_p)
            n_exact += check(t, ra)
    if orc:
        print("oracle matches the reference for %d steps (bit-exact float32 observations on %d of them)" % (args.steps, n_exact))
    meta = dict(kwargs=kwargs, seed=args.seed, n_steps=args.steps)
    if multi_episode:
        meta.update(variant=args.variant, reset_at_done=True)
    out = {"meta_json": np.array(json.dumps(meta))}
    out["act_a"] = np.stack(acts_a).astype(np.int8)
    out["act_p"] = np.array(acts_p, np.int8)
    for k, v in rec.items():
        if k in ("rew_a", "rew_p", "done"):
            out[k] = np.stack(v)          # steps 1..N
        else:
            out[k] = np.stack(v)          # steps 0..N
    path = variant_path(args.variant) if multi_episode else os.path.join(OUT, "%s.npz" % (args.name or "covid_seed%d" % args.seed))
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, **out)
    print(path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
