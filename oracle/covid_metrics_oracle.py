"""TEST INFRASTRUCTURE ONLY — numpy restatement of the COVID-19 episode metrics the device computes.

Restates aie_covid_metrics_kernel over the accumulators the step kernel keeps (covid_step_env's STATS,
covid_metrics_row in ai_economist_b200/csrc/aie_covid_core.cuh), column for column in the kernel's order.  Its inputs
are the float32 records the device stored, not oracle/covid_oracle.py's own trajectory: the kernel matches the
reference to 1e-6 relative, so this restatement is what the device is held to bit for bit (tests/test_covid_metrics.py).
"""
import numpy as np

F32 = np.float32


def _cv_pow(x, e):   # the kernel's cv_pow: numpy's scalar-exponent fast paths, powf otherwise
    x, e = F32(x), F32(e)
    if e == F32(-1):
        return F32(1) / x
    if e == F32(2):
        return x * x
    if e == F32(0.5):
        return np.sqrt(x)
    if e == F32(1):
        return x
    if e == F32(0):
        return F32(1)
    return np.power(x, e)


def _cv_crra(x, eta):
    ax = F32(365) * F32(x)
    axc = np.minimum(np.maximum(ax, F32(0.1)), F32(3))
    one_m = F32(1) - F32(eta)
    return (F32(1) + (_cv_pow(axc, one_m) - F32(1)) / one_m) / F32(365)


def _cv_minmax(x, lo, hi):
    return (F32(x) - F32(lo)) / ((F32(hi) - F32(lo)) + F32(1e-10))


def covid_metric_accumulators(p, records):
    """The step kernel's accumulators after the steps of one episode: records = the float32 state records [9, S]
    (susceptible .. postsubsidy, the stepper's "state" buffer of one replica) at t = 0 (the reset) .. t_now.
    Returns (sums float64 [4, S]: Unemployed, Stringency Level, Postsubsidy Productivity, Subsidy; index float32
    [2, S + 1]: health then economic index of each state then the planner)."""
    S = p["n_states"]
    sums = np.zeros((4, S), np.float64)
    index = np.zeros((2, S + 1), np.float32)
    vol = np.float64(p["value_of_life"])
    for t in range(1, len(records)):
        r, q = np.asarray(records[t], F32), np.asarray(records[t - 1], F32)
        for k, row in enumerate((5, 6, 8, 7)):
            sums[k] += r[row].astype(np.float64)
        md = r[3] - q[3]
        post, sub = r[8], r[7]
        for a in range(S):
            h = F32((np.float64(-md[a]) * vol) / np.float64(p["agents_health_norm"][a]))
            h = _cv_minmax(h, p["min_marginal_agent_health_index"][a], p["max_marginal_agent_health_index"][a])
            ec = _cv_crra(post[a] / F32(p["agents_economic_norm"][a]), p["crra_eta"])
            ec = _cv_minmax(ec, p["min_marginal_agent_economic_index"][a], p["max_marginal_agent_economic_index"][a])
            index[0, a] = index[0, a] + h
            index[1, a] = index[1, a] + ec
        sum_md, sum_sub, sum_post = np.sum(md), np.sum(sub), np.sum(post)   # numpy's float32 pairwise sums
        ph = (np.float64(-sum_md) * vol) / np.float64(p["planner_health_norm"])
        lo, hi = F32(p["min_marginal_planner_health_index"]), F32(p["max_marginal_planner_health_index"])
        ph = (ph - np.float64(lo)) / np.float64((hi - lo) + F32(1e-10))
        cost = (F32(1) + F32(p["risk_free_interest_rate"])) * sum_sub
        pe = _cv_crra((sum_post - cost) / F32(p["planner_economic_norm"]), p["crra_eta"])
        pe = _cv_minmax(pe, p["min_marginal_planner_economic_index"], p["max_marginal_planner_economic_index"])
        index[0, S] = F32(np.float64(index[0, S]) + ph)
        index[1, S] = index[1, S] + pe
    return sums, index


def covid_metrics_row(p, end, sums, index):
    """One row of aie_covid_episode_metrics: end = float32 [4, S] I, R, D, V; sums / index as covid_metric_accumulators.
    Columns: 8 per state, then 7 usa/ (aie_covid_get_metric_layout)."""
    S, T, us_pop = p["n_states"], np.float64(p["episode_length"]), np.float64(p["us_population"])
    end = np.asarray(end, F32)
    row = np.zeros(8 * S + 7, np.float64)
    for a in range(S):
        r = row[8 * a: 8 * a + 8]
        for k in range(3):
            r[k] = np.float64(np.int32(end[k, a])) / 1e6
        r[3] = ((sums[0, a] / T) / np.float64(p["population"][a])) * 100.0
        r[4] = sums[1, a] / T
        r[5] = sums[2, a] / 1e9
        r[6], r[7] = np.float64(index[0, a]), np.float64(index[1, a])
    v = d = u = sub = post = np.float64(0)
    for a in range(S):   # sequential, in state order
        v += np.float64(end[3, a]); d += np.float64(end[2, a])
        u += sums[0, a]; sub += sums[3, a]; post += sums[2, a]
    row[8 * S:] = [(v / us_pop) * 100.0, d / 1e3, ((u / us_pop) / T) * 100.0, sub / 1e12, post / 1e12,
                   np.float64(index[0, S]), np.float64(index[1, S])]
    return row
