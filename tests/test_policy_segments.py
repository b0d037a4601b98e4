"""The policy sampler, `evaluate_actions` and the random policy at every 32-entry chunk of a mask segment, with the edge
cases planted at chosen lanes and chunks.

The device code works one mask segment per warp, in up to five 32-entry chunks (MAX_MASK = 160); the host build of the
same source walks the segment serially.  These tests build configs whose segments end on either side of every chunk
boundary (33 ... 160 entries), write masks, logits and stored actions directly, and hold both builds to the numpy
restatements of tests/test_policy_sampler.py (`draw`) and tests/test_evaluate_actions.py (`ref_segment`), and CUDA to
the host build on identical inputs.  Out-of-range stored actions are planted only away from the first and last segment
of a tensor, so that even a wrong kernel reads nothing outside it."""
import math

import numpy as np
import pytest
import torch

from ai_economist_b200 import _abi, foundation
from ai_economist_b200.workloads import COVID_KWARGS, covid_reference_config
from tests.test_evaluate_actions import check_all
from tests.test_policy_sampler import (as_f32, call_stream, check_segment, env_key, gtb_segments, make_env, to_bf16_bits,
                                       uniform)

POS = (0, 1, 30, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 158, 159)
P_KINDS = ("only", "max_at", "pair", "tie", "nan_open", "inf_open", "nan_closed", "inf_closed", "flt_max", "underflow",
           "mask_values", "act_closed")
I_KINDS = ("equal", "all_ninf", "none_open", "act_n", "act_neg")   # one plan per length: p does not matter
FLT_MAX, BF16_MAX = float(np.finfo(np.float32).max), float(np.uint32(0x7F7F0000).view(np.float32))

# ---------------------------------------------------------------------------------------------- configs
_15 = dict(scenario_name="layout_from_file/simple_wood_and_stone", env_layout_file="env-pure_and_mixed-15x15.txt",
           n_agents=3, world_size=[15, 15], episode_length=20, multi_action_mode_agents=False,
           multi_action_mode_planner=True, flatten_observations=True, flatten_masks=True, fixed_four_skill_and_loc=False,
           starting_agent_coin=5)


def cda(m, multi=False):
    return dict(_15, components=[("ContinuousDoubleAuction", dict(max_bid_ask=m, max_num_orders=3)), ("Gather", {})],
                multi_action_mode_agents=multi)


def tax(rate_disc, n_brackets=3, multi=True):
    return dict(_15, components=[("ContinuousDoubleAuction", dict(max_num_orders=3)), ("Gather", {}),
                                 ("PeriodicBracketTax", dict(bracket_spacing="linear", n_brackets=n_brackets, period=5,
                                                             rate_disc=rate_disc, tax_model="model_wrapper"))],
                multi_action_mode_planner=multi)


# name -> (kwargs over c1_tutorial's, or a config of test_policy_sampler, or the COVID-19 subsidy levels; the segment
# lengths it must reach)
GTB = {
    "cda6": (cda(6), {33}), "cda14": (cda(14), {65}), "cda22": (cda(22), {97}), "cda30": (cda(30), {129}),
    "cda31": (cda(31), {133}), "cda31_multi": (cda(31, multi=True), {33}),
    "bracket30": (tax(1 / 30), {32}), "bracket31": (tax(1 / 31), {33}), "bracket62": (tax(1 / 62), {64}),
    "bracket63": (tax(1 / 63), {65}),
    "single160": (tax(1 / 52, multi=False), {160}), "single129": (tax(1 / 63, n_brackets=2, multi=False), {129}),
    "one_step": (None, {101}), "tax_single_planner": (None, {148}),
}
COVID = {"covid%d" % L: L for L in (30, 31, 32, 63, 64, 95, 96, 127, 128, 158, 159)}
CFGS = list(GTB) + list(COVID)


def _make(cfg, n_envs, factory, obs_dtype):
    if cfg in COVID:
        kw = covid_reference_config(dict(COVID_KWARGS, num_subsidy_levels=COVID[cfg]))
        name = kw.pop("scenario_name")
        dev = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
        env = foundation.make_env_instance(name, n_envs=n_envs, auto_reset=True, obs_dtype=obs_dtype, **dev, **kw)
        env.reset()
        return env
    over = GTB[cfg][0]
    return make_env(cfg, n_envs, factory, obs_dtype) if over is None else make_env("c1_tutorial", n_envs, factory,
                                                                                  obs_dtype, **over)


def emu_factory_of(cfg):
    from tests.emu.emu_stepper import emu_factory
    from tests.test_covid_obs_bf16 import emu
    return (lambda params, n, ar, obs_dtype=None: emu(params, n, ar, obs_dtype=obs_dtype)) if cfg in COVID else emu_factory


# ---------------------------------------------------------------------------------------------- segments of a row
class Seg:
    """One mask segment of a row: where its mask, logits and action sit (index tuples after the row), its length, and
    the sampler's key of it from the env key k."""

    def __init__(self, who, mi, li, ai, n, key):
        self.who, self.mi, self.li, self.ai, self.n, self.key = who, mi, li, ai, n, key


def row_segments(env, covid):
    if covid:
        S = env.n_agents
        segs = [Seg("a", (slice(None), s), (s, slice(None)), (s,), 1 + env.stepper.p["num_stringency_levels"],
                    lambda k, s=s: k + 0x100 * s) for s in range(S)]
        return segs + [Seg("p", (slice(None),), (slice(None),), (), 1 + env.stepper.p["num_subsidy_levels"],
                           lambda k: k ^ 0xABCDEF)]
    out = []
    for who, unit, slot, off, ln, ko in gtb_segments(env.spec, env.stepper.dims):
        sl = slice(off, off + ln)
        mi = (unit, sl) if who == "a" else (sl,)
        out.append(Seg(who, mi, mi, (unit, slot) if who == "a" else (slot,), ln, lambda k, ko=ko: k + ko))
    return out


def lengths(segs):
    return sorted({s.n for s in segs})


def positions(n):
    return [p for p in POS if p < n]


def plans_of(n):
    ps = positions(n)
    return [(k, p) for k in P_KINDS for p in ps] + [(k, ps[0]) for k in I_KINDS]


def rows_needed(segs):
    """Rows 1 .. E-2 carry the plans (rows 0 and E-1, the first and last of every tensor, stay random)."""
    return 2 + max(math.ceil(len(plans_of(n)) / sum(s.n == n for s in segs)) for n in lengths(segs))


def batch_size(segs, units, at_least=0):
    """Planted rows plus the two random ones, chosen so that neither launch shape's warp count is a multiple of 8."""
    E = max(rows_needed(segs), at_least)
    while E % 8 == 0 or (E * units) % 8 == 0:
        E += 1
    return E


def partner(p, n):
    """An entry in another 32-entry chunk than p where there is one (both listed lanes when they fit)."""
    other = [q for q in positions(n) if q // 32 != p // 32]
    if other:
        return min(other, key=lambda q: (q < p, abs(q - p)))
    return n - 1 if p != n - 1 else 0


def plant(kind, n, p, rng, bf16_logits):
    """(mask, logits, stored-action override or None) of one planted segment, in float32."""
    m = (rng.random_sample(n) < 0.8).astype(np.float32)
    l = (rng.standard_normal(n) * 3).astype(np.float32)
    act = None
    big = BF16_MAX if bf16_logits else FLT_MAX
    nb = [j for j in (p - 1, p + 1, p + 2, p + 3, p + 4, p + 5) if 0 <= j < n]
    if kind == "only":
        m[:] = 0.0
        m[p] = 1.0
    elif kind == "equal":
        m[:], l[:] = 1.0, 0.75
    elif kind == "max_at":
        m[:], l[:] = 1.0, -np.inf
        l[p] = rng.standard_normal()
    elif kind in ("pair", "tie"):
        a, b = sorted((p, partner(p, n)))
        if kind == "pair":
            m[:] = 0.0
            l[a] = l[b] = 1.25
        else:
            l[a] = l[b] = l.max() + 1.0
        m[a] = m[b] = 1.0
    elif kind in ("nan_open", "inf_open", "nan_closed", "inf_closed"):
        m[p] = 1.0 if kind.endswith("open") else 0.0
        l[p] = np.nan if kind.startswith("nan") else np.inf
        if nb:
            m[nb[0]] = 1.0
    elif kind == "all_ninf":
        l[:] = -np.inf
        m[p] = 1.0
    elif kind == "none_open":
        m[:] = 0.0
    elif kind == "flt_max":
        m[p], l[p] = 1.0, big
        for j in nb[:2]:
            m[j], l[j] = 1.0, -big
    elif kind == "underflow":
        m[:] = 1.0
        if nb:
            rest = np.delete(l, [p, nb[0]])
            top = float(rest.max()) if len(rest) else 0.0
            l[p], l[nb[0]] = top - 750.0, top - 740.0   # weight 0, and a subnormal weight, in float64
        else:
            l[p] = -750.0
    elif kind == "mask_values":
        m[p] = -0.0
        for j, v in zip(nb, (1e-45, 0.5, -1.0, np.nan, 2.0 ** -133)):   # 2^-133: bfloat16 bits 0x0001
            m[j] = v
    elif kind == "act_closed":
        m[p], act = 0.0, p
    elif kind == "act_n":
        act = n
    elif kind == "act_neg":
        act = -1
    return m, l, act


def random_segment(n, rng):
    m = (rng.random_sample(n) < 0.8).astype(np.float32)
    l = (rng.standard_normal(n) * 3).astype(np.float32)
    l[rng.random_sample(n) < 0.1] = -np.inf
    return m, l


class Batch:
    """Planted inputs of E rows: float32 masks and logits (agent, planner), the plans per (row, segment), and the
    stored-action overrides of the evaluator."""

    def __init__(self, env, segs, E, seed, bf16_logits, n_random=0):
        rng = np.random.RandomState(seed)
        st = env.stepper
        shp = lambda name: tuple(st.buf[name].shape[1:])
        self.M = {"a": np.zeros((E,) + shp("mask_agent"), np.float32), "p": np.zeros((E,) + shp("mask_planner"), np.float32)}
        sa, sp = st._policy_shapes()[:2]
        self.L = {"a": np.zeros((E,) + tuple(sa[1:]), np.float32),
                  "p": None if sp is None else np.zeros((E,) + tuple(sp[1:]), np.float32)}
        self.plan, self.acts, self.segs, self.E = {}, {}, segs, E
        self.rows = {0, E - 1} | set(int(r) for r in rng.choice(E, min(E, n_random), replace=False))
        todo = {n: plans_of(n) for n in lengths(segs)}
        for r in range(E):
            for i, s in enumerate(segs):
                if 0 < r < E - 1 and todo[s.n]:
                    kind, p = todo[s.n].pop(0)
                    m, l, act = plant(kind, s.n, p, rng, bf16_logits)
                    self.plan[r, i] = (kind, p)
                    if act is not None:
                        self.acts[r, i] = act
                else:
                    m, l = random_segment(s.n, rng)
                self.M[s.who][(r,) + s.mi] = m
                self.L[s.who][(r,) + s.li] = l
        assert not any(todo.values()), "too few rows for the plans"

    def checked(self, e, i):
        """Segments held to the restatements: every planted one, and every segment of the random rows."""
        return (e, i) in self.plan or e in self.rows

    def kinds_by_length(self):
        out = {}
        for (r, i), (kind, _) in self.plan.items():
            out.setdefault(self.segs[i].n, set()).add(kind)
        return out


def stored(x, bf16):
    """float32 values in a tensor's storage: float32, or bfloat16 bits (round to nearest even)."""
    return None if x is None else (to_bf16_bits(x) if bf16 else np.ascontiguousarray(x, np.float32))


# ---------------------------------------------------------------------------------------------- backends
class Side:
    """One env (CUDA or the host build) and conversions between its buffers and numpy."""

    def __init__(self, env):
        self.env, self.st = env, env.stepper
        self.cuda = not isinstance(self.st.buf["mask_agent"], np.ndarray)

    def dev(self, x):
        if x is None or not self.cuda:
            return x
        if x.dtype == np.uint16:
            return torch.from_numpy(x.view(np.int16)).view(torch.bfloat16).cuda()
        return torch.from_numpy(np.ascontiguousarray(x)).cuda()

    def np(self, x):
        if x is None or isinstance(x, np.ndarray):
            return x
        x = x.detach()
        return x.view(torch.int16).cpu().numpy().view(np.uint16) if x.dtype == torch.bfloat16 else x.cpu().numpy()

    def put_masks(self, ma, mp):
        for name, x in (("mask_agent", ma), ("mask_planner", mp)):
            buf = self.st.buf[name]
            if self.cuda:
                buf.copy_(self.dev(x))
            else:
                buf[...] = x

    def sample(self, la, lp, seed, greedy):
        lpa, lpp = self.env.sample_actions(self.dev(la), self.dev(lp), seed=seed, greedy=greedy)
        b = self.st.buf
        return (self.np(b["actions_agent"]).copy(), self.np(b["actions_planner"]).copy(), self.np(lpa).copy(),
                None if lpp is None else self.np(lpp).copy())

    def evaluate(self, la, lp, acts, masks):
        d = lambda x: None if x is None else self.dev(np.ascontiguousarray(x))
        res = self.st.evaluate_policy(d(la), d(lp), (d(acts[0]), d(acts[1])), (d(masks[0]), d(masks[1])))
        return [self.np(x) for x in res]

    def backward(self, la, lp, acts, masks, glp, gh):
        d = lambda x: None if x is None else self.dev(np.ascontiguousarray(x))
        g = self.st.evaluate_policy_backward(d(la), d(lp), (d(acts[0]), d(acts[1])), (d(masks[0]), d(masks[1])),
                                             (d(glp[0]), d(glp[1])), (d(gh[0]), d(gh[1])))
        return [self.np(x) for x in g]


def planner_on(side):
    return side.st._policy_shapes()[1] is not None


# ---------------------------------------------------------------------------------------------- one run
def run_planted(side, B, mask_bf16, logit_bf16, seed=77, twin=None):
    """Sampler (three stochastic calls, one greedy) and evaluator on B's inputs.  Holds B's checked segments to the
    restatements and, with a twin (the host build on the same inputs), every row of both to each other.  Returns the
    counters the callers assert on."""
    planner = planner_on(side)
    ma, mp = stored(B.M["a"], mask_bf16), stored(B.M["p"], mask_bf16)
    la, lp = stored(B.L["a"], logit_bf16), stored(B.L["p"], logit_bf16) if planner else None
    ma32, mp32, la32, lp32 = as_f32(ma), as_f32(mp), as_f32(la), as_f32(lp)
    rows = sorted({r for r, _ in B.plan} | B.rows)
    sides = [side] + ([twin] if twin else [])
    for s in sides:
        s.put_masks(ma, mp)
    cnt = dict(draws=0, near=0, pair=0, pair_low=0)
    calls = []
    for call, greedy in enumerate((False, False, False, True), start=1):
        outs = [s.sample(la, lp, seed, greedy) for s in sides]
        if twin:   # CUDA against the host build: actions byte-equal, log-probabilities within one float32 ulp
            (a1, p1, l1, q1), (a2, p2, l2, q2) = outs
            assert a1.tobytes() == a2.tobytes() and p1.tobytes() == p2.tobytes()
            assert _close_lp(l1, l2) and (q1 is None or _close_lp(q1, q2))
        aa, ap, lpa, lpp = outs[0]
        s_key = call_stream(seed, call)
        for r in rows:
            k = env_key(s_key, r)
            for i, sg in enumerate(B.segs):
                if not B.checked(r, i):
                    continue
                o = (ma32 if sg.who == "a" else mp32)[(r,) + sg.mi] != 0
                l = (la32 if sg.who == "a" else lp32)[(r,) + sg.li]
                act = (aa if sg.who == "a" else ap)[(r,) + sg.ai]
                got_lp = (lpa if sg.who == "a" else lpp)[(r,) + sg.ai]
                cnt["near"] += check_segment(o, l, uniform(sg.key(k)), greedy, act, got_lp)
                cnt["draws"] += 1
                if not greedy and B.plan.get((r, i), ("",))[0] == "pair":
                    cnt["pair"] += 1
                    cnt["pair_low"] += int(act == min(np.nonzero(o)[0]))
                if greedy and B.plan.get((r, i), ("",))[0] == "tie":
                    assert int(act) == int(np.nonzero(o & (l == l[o].max()))[0][0])
        calls.append((aa, ap, lpa, lpp))
    # the evaluator on [T, E] rows: call 1 (stochastic) and call 4 (greedy), the planted stored actions substituted
    T = 2
    st_a = np.stack([calls[0][0], calls[3][0]])
    st_p = np.stack([calls[0][1], calls[3][1]]) if planner else None
    bad = np.zeros(st_a.shape[:2] + (len(B.segs),), bool)
    for (r, i), act in B.acts.items():
        sg = B.segs[i]
        (st_a if sg.who == "a" else st_p)[(slice(None), r) + sg.ai] = act
        bad[:, r, i] = True
    rep = lambda x: None if x is None else np.ascontiguousarray(np.stack([x] * T))
    X = dict(la=rep(la), lp=rep(lp), ma=rep(ma), mp=rep(mp), aa=st_a, ap=st_p)
    res = side.evaluate(X["la"], X["lp"], (X["aa"], X["ap"]), (X["ma"], X["mp"]))
    assert res[0].shape == st_a.shape and res[0].dtype == np.float32
    # log-probabilities of the sampler's own actions: its own bits
    for t, c in enumerate((0, 3)):
        for sg_i, sg in enumerate(B.segs):
            got = (res[0] if sg.who == "a" else res[1])[(t, slice(None)) + sg.ai]
            want = (calls[c][2] if sg.who == "a" else calls[c][3])[(slice(None),) + sg.ai]
            keep = ~bad[t, :, sg_i]
            assert got[keep].tobytes() == want[keep].tobytes()
    if twin:
        res2 = twin.evaluate(X["la"], X["lp"], (X["aa"], X["ap"]), (X["ma"], X["mp"]))
        for x, y in zip(res, res2):
            assert (x is None and y is None) or _close_lp(x, y)
    F32 = _flat({k: as_f32(v) for k, v in X.items()})
    n, kinds = check_all(lambda r: _views(B, F32, r, r % B.E), (T, B.E), res)
    cnt["kinds"] = kinds
    # a gathered minibatch: every checked row of t = 1, then of t = 0 in reverse
    idx = np.r_[[B.E + r for r in rows], [r for r in rows][::-1]]
    G = {k: (None if v is None else np.ascontiguousarray(v.reshape((-1,) + v.shape[2:])[idx])) for k, v in X.items()}
    G32 = {k: as_f32(v) for k, v in G.items()}
    N = len(idx)
    gres = side.evaluate(G["la"], G["lp"], (G["aa"], G["ap"]), (G["ma"], G["mp"]))
    for x, y in zip(gres, res):
        if x is not None:
            assert x.tobytes() == y.reshape((-1,) + y.shape[2:])[idx].tobytes()
    gviews = lambda r: _views(B, G32, r, int(idx[r]) % B.E)
    rng = np.random.RandomState(5)
    up = lambda like: None if like is None else (rng.standard_normal(like.shape) * 2).astype(np.float32)
    for mode in ("lp", "h", "both"):
        glp = (up(gres[0]), up(gres[1])) if mode != "h" else (None, None)
        gh = (up(gres[2]), up(gres[3])) if mode != "lp" else (None, None)
        ga, gp = side.backward(G["la"], G["lp"], (G["aa"], G["ap"]), (G["ma"], G["mp"]), glp, gh)
        assert ga.shape == G["la"].shape and ga.dtype == G["la"].dtype
        check_all(gviews, (N,), gres, grads=(ga, gp), ups=(glp[0], glp[1], gh[0], gh[1]), bf16=logit_bf16)
        if twin:   # within one ulp of the host build plus 1e-12 times the upstream gradient
            ha, hp = twin.backward(G["la"], G["lp"], (G["aa"], G["ap"]), (G["ma"], G["mp"]), glp, gh)
            for x, y, who in ((ga, ha, "a"), (gp, hp, "p")):
                if x is not None:
                    assert _close_grad_rows(as_f32(x), as_f32(y), who, glp, gh, logit_bf16)
    cnt["segments"] = n
    return cnt


def _views(B, F, r, e):
    """check_all's views of B's checked segments of flat row r (env row e) of the flat float32 inputs F."""
    for i, sg in enumerate(B.segs):
        if not B.checked(e, i):
            continue
        M, L, A = (F["ma"], F["la"], F["aa"]) if sg.who == "a" else (F["mp"], F["lp"], F["ap"])
        if sg.who == "a":
            unit, slot = (sg.ai[0], sg.ai[1]) if len(sg.ai) == 2 else (sg.ai[0], None)
        else:
            unit, slot = 0, (sg.ai[0] if sg.ai else None)
        off = sg.mi[-1].start if slot is not None else None
        yield M[r][sg.mi] != 0, L[r][sg.li], int(A[r][sg.ai]), (sg.who, unit, slot, off, sg.n)


def _flat(X):
    return {k: (None if v is None else v.reshape((-1,) + v.shape[2:])) for k, v in X.items()}


def _close_lp(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(np.all((np.abs(a - b) <= np.spacing(np.abs(b))) | (np.isnan(a) & np.isnan(b))))


def _close_grad_rows(x, y, who, glp, gh, bf16):
    """Within one ulp of the output dtype plus 1e-12 times the largest upstream gradient (NaN where the other is NaN)."""
    ulp = np.spacing(np.abs(y)) * (2.0 ** 16 if bf16 else 1.0)
    scale = 0.0
    for u in (glp[0 if who == "a" else 1], gh[0 if who == "a" else 1]):
        if u is not None:
            scale += float(np.abs(u).max())
    return bool(np.all((np.abs(x.astype(np.float64) - y) <= ulp + 1e-12 * scale) | (np.isnan(x) & np.isnan(y))))


# ---------------------------------------------------------------------------------------------- CPU (host build)
def _expected(cfg):
    return {11, 1 + COVID[cfg]} if cfg in COVID else GTB[cfg][1]


def _planted(cfg, factory, mask_bf16, logit_bf16, at_least=0, n_random=0, seed=3):
    """An env of cfg sized for every plan of its segment lengths, and its planted batch."""
    covid = cfg in COVID
    probe = _make(cfg, 1, emu_factory_of(cfg), None)
    segs = row_segments(probe, covid)
    assert _expected(cfg) <= set(lengths(segs)), (cfg, lengths(segs))
    E = batch_size(segs, len(segs), at_least)
    env = _make(cfg, E, factory, torch.bfloat16 if mask_bf16 else None)
    return env, Batch(env, segs, E, seed, logit_bf16, n_random)


def _assert_counts(B, cnt, cfg):
    assert cnt["draws"] > 0 and cnt["near"] == 0
    for n, kinds in B.kinds_by_length().items():   # every planted kind at every length
        assert kinds == set(P_KINDS) | set(I_KINDS), (cfg, n, set(P_KINDS) | set(I_KINDS) - kinds)
    assert _expected(cfg) <= set(B.kinds_by_length())
    k = cnt["kinds"]
    assert k["closed"] >= 1 and k["bad"] >= 3 and k["bad_action"] >= 3 and k["ninf_open"] >= 1
    # two open entries of equal logits: each drawn half the time (binomial, three stochastic calls)
    from scipy import stats
    assert cnt["pair"] >= 3 and stats.binomtest(cnt["pair_low"], cnt["pair"], 0.5).pvalue > 1e-4


DTYPES = [(False, False), (True, True), (False, True)]   # (bfloat16 masks, bfloat16 logits)


@pytest.mark.parametrize("cfg", CFGS)
def test_emulated_planted_segments(cfg):
    """Every segment length of the table, every planted kind at every listed lane: the host build's sampler and
    evaluator against the restatements, float32 and bfloat16 masks and logits."""
    for mask_bf16, logit_bf16 in DTYPES if cfg in ("cda31", "single160", "covid159") else DTYPES[:2]:
        env, B = _planted(cfg, emu_factory_of(cfg), mask_bf16, logit_bf16)
        cnt = run_planted(Side(env), B, mask_bf16, logit_bf16)
        _assert_counts(B, cnt, cfg)


@pytest.mark.parametrize("cfg", ["cda31", "single160", "covid159"])
def test_emulated_extreme_stored_actions(cfg):
    """INT_MAX and INT_MIN as stored actions (host build only): log-probability NaN, the entropy as usual, the open
    entries' gradient NaN and the closed ones 0."""
    env, B = _planted(cfg, emu_factory_of(cfg), False, False)
    side, planner = Side(env), planner_on(Side(env))
    ma, mp, la, lp = B.M["a"], B.M["p"], B.L["a"], (B.L["p"] if planner else None)
    side.put_masks(ma, mp)
    aa, ap, _, _ = side.sample(la, lp, 5, False)
    ref = side.evaluate(la, lp, (aa, ap), (ma, mp))
    for v in (np.iinfo(np.int32).max, np.iinfo(np.int32).min):
        xa, xp = aa.copy(), (ap.copy() if planner else None)
        sg = B.segs[-1]
        (xa if sg.who == "a" else xp)[(slice(None),) + sg.ai] = v
        res = side.evaluate(la, lp, (xa, xp), (ma, mp))
        got = (res[0] if sg.who == "a" else res[1])[(slice(None),) + sg.ai]
        h, h0 = [(x[2] if sg.who == "a" else x[3])[(slice(None),) + sg.ai] for x in (res, ref)]
        opened = np.array([B.M[sg.who][(r,) + sg.mi].astype(bool).any() for r in range(B.E)])
        assert np.isnan(got[opened]).all() and (got[~opened] == 0).all()
        assert h.tobytes() == h0.tobytes()
        ones = lambda x: None if x is None else np.ones(x.shape, np.float32)
        ga, gp = side.backward(la, lp, (xa, xp), (ma, mp), (ones(xa), ones(xp)), (None, None))
        g = ga if sg.who == "a" else gp
        for r in range(B.E):
            gr, o = g[(r,) + sg.li], B.M[sg.who][(r,) + sg.mi] != 0
            if o.any() and not np.isnan(h[r]):
                assert np.isnan(gr[o]).all()
            assert (gr[~o] == 0).all()


@pytest.mark.parametrize("cfg", ["cda31", "cda31_multi", "single160", "single129", "one_step"])
def test_emulated_random_policy_draws_open_entries(cfg):
    """sample_random_actions on the planted masks: an open entry of every segment with one (the only one where a
    single entry is open, chunk 4 included), 0 where nothing is open, and every full chunk of an all-open segment
    reached."""
    env, B = _planted(cfg, emu_factory_of(cfg), False, False)
    side = Side(env)
    side.put_masks(B.M["a"], B.M["p"])
    seen = {}
    for _ in range(60):   # one seed: the call counter moves the stream (seed == call would repeat it)
        side.st.sample_random_actions(seed=7)
        acts = {w: side.np(side.st.buf["actions_agent" if w == "a" else "actions_planner"]) for w in "ap"}
        for r in range(B.E):
            for i, sg in enumerate(B.segs):
                o = B.M[sg.who][(r,) + sg.mi] != 0
                a = int(acts[sg.who][(r,) + sg.ai])
                kind, p = B.plan.get((r, i), ("", None))
                assert (0 <= a < sg.n and o[a]) if o.any() else a == 0, (cfg, r, i, kind, a)
                if kind == "only":
                    assert a == p
                if kind == "equal":
                    seen.setdefault((r, i), set()).add(a // 32)
    for (r, i), chunks in seen.items():   # 60 uniform draws miss a full chunk of 160 entries with odds 0.8^60
        assert chunks >= set(range(B.segs[i].n // 32)), (r, i, chunks)


def _covid_levels(L, factory):
    kw = covid_reference_config(dict(COVID_KWARGS, num_subsidy_levels=L))
    name = kw.pop("scenario_name")
    dev = dict(stepper_factory=factory) if factory else dict(device="cuda:0")
    env = foundation.make_env_instance(name, n_envs=3, auto_reset=True, **dev, **kw)
    env.reset()
    return env


def check_refusals(factory_covid, factory_gtb, to_dev):
    """COVID-19: 159 subsidy levels sample and evaluate, 160 are refused by both before any launch.  Gather-trade-build:
    a single-action planner of 1 + 3 x 53 = 160 entries is created, one of 1 + 3 x 54 = 163 is refused."""
    for L, ok in ((159, True), (160, False)):
        env = _covid_levels(L, factory_covid)
        st = env.stepper
        sa, sp = st._policy_shapes()[:2]
        la, lp = to_dev(np.zeros(sa, np.float32)), to_dev(np.zeros(sp, np.float32))
        acts = (st.buf["actions_agent"], st.buf["actions_planner"])
        masks = (st.buf["mask_agent"], st.buf["mask_planner"])
        n0 = st.launch_count()
        if ok:
            env.sample_actions(la, lp, seed=1)
            st.evaluate_policy(la, lp, acts, masks)
            continue
        with pytest.raises(_abi.AieError, match="more than 159 subsidy levels"):
            env.sample_actions(la, lp, seed=1)
        with pytest.raises(_abi.AieError, match="more than 159 subsidy levels"):
            st.evaluate_policy(la, lp, acts, masks)
        with pytest.raises(_abi.AieError, match="more than 159 subsidy levels"):
            st.evaluate_policy_backward(la, lp, acts, masks)
        assert st.launch_count() == n0
    env = make_env("c1_tutorial", 2, factory_gtb, None, **tax(1 / 52, multi=False))
    assert env.stepper.dims.mask_planner == 160
    with pytest.raises(_abi.AieError, match="single-action planner mask too long"):
        make_env("c1_tutorial", 2, factory_gtb, None, **tax(1 / 53, multi=False))


def test_emulated_refusals_at_160():
    from tests.emu.emu_stepper import emu_factory
    check_refusals(emu_factory_of("covid159"), emu_factory, lambda x: x)


# ---------------------------------------------------------------------------------------------- GPU
def _cuda_and_twin(cfg, mask_bf16, logit_bf16, at_least=0, n_random=4):
    env, B = _planted(cfg, None, mask_bf16, logit_bf16, at_least=at_least, n_random=n_random)
    twin = _make(cfg, B.E, emu_factory_of(cfg), torch.bfloat16 if mask_bf16 else None)
    return Side(env), Side(twin), B


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CFGS)
def test_cuda_planted_segments(cfg, monkeypatch):
    """The CUDA sampler and evaluator on the planted batches: against the restatements, and against the host build on
    every row; gather-trade-build configs in both launch shapes (one warp per env or row, one per unit)."""
    for mask_bf16, logit_bf16 in DTYPES:
        for per_unit in ((None,) if cfg in COVID else ("0", "1")):
            if per_unit is not None:
                monkeypatch.setenv("AIE_POLICY_PER_UNIT", per_unit)
            cuda, twin, B = _cuda_and_twin(cfg, mask_bf16, logit_bf16)
            _assert_counts(B, run_planted(cuda, B, mask_bf16, logit_bf16, twin=twin), cfg)
            del cuda
            torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["single160", "cda31", "covid159"])
def test_cuda_large_batch(cfg):
    """About 2 048 rows, so that the grid spans many CTAs: every planted row and 24 random ones against the
    restatements, every row against the host build."""
    cuda, twin, B = _cuda_and_twin(cfg, False, False, at_least=2048, n_random=24)
    assert B.E > 2048
    _assert_counts(B, run_planted(cuda, B, False, False, twin=twin), cfg)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["cda30", "cda31", "cda31_multi", "bracket63", "single160", "single129", "one_step",
                                 "covid159"])
def test_cuda_random_policy_matches_host_build(cfg):
    """sample_random_actions on the planted masks (among them every entry open, and one open entry in each listed lane,
    chunk 4 included): CUDA's actions byte-equal to the host build's."""
    cuda, twin, B = _cuda_and_twin(cfg, False, False)
    kinds = B.kinds_by_length()
    assert all({"equal", "only"} <= k for k in kinds.values())
    for s in (cuda, twin):
        s.put_masks(B.M["a"], B.M["p"])
    for _ in range(3):
        got = []
        for s in (cuda, twin):
            s.st.sample_random_actions(seed=7)
            got.append([s.np(s.st.buf[k]).tobytes() for k in ("actions_agent", "actions_planner")])
        assert got[0] == got[1]


@pytest.mark.gpu
def test_cuda_refusals_at_160():
    check_refusals(None, None, lambda x: torch.from_numpy(x).cuda())
