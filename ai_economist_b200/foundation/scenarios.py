"""Scenario classes: constructor kwargs (same names/defaults as the reference) and the HOST-side reset.

Reset stays on the host in this round (SURVEY §8f row 1): it draws from a per-env numpy legacy RandomState in
exactly the reference's order, so a seeded env starts from the reference's state and RNG position; the
post-reset snapshot is uploaded through aie_load_state.  The per-step scenario logic (resource regeneration,
observations, rewards) runs on the GPU.

reference: scenarios/simple_wood_and_stone/layout_from_file.py:24-650, dynamic_layout.py:27-700
"""
import os

import numpy as np

from .registrar import Registry

MAP_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "map_txt")
_SWF = {"coin_eq_times_productivity": 0, "inv_income_weighted_coin_endowments": 1, "inv_income_weighted_utility": 2}


class BaseScenario:
    """Scenario-level kwargs shared by the simple_wood_and_stone family."""
    name = ""
    agent_subclasses = ["BasicMobileAgent", "BasicPlanner"]
    required_entities = []

    def __init__(self, env, planner_gets_spatial_info=True, full_observability=False,
                 mobile_agent_observation_range=5, starting_agent_coin=0, isoelastic_eta=0.23, energy_cost=0.21,
                 energy_warmup_constant=0, energy_warmup_method="decay",
                 planner_reward_type="coin_eq_times_productivity", mixing_weight_gini_vs_coin=0.0):
        self.env = env
        self.planner_gets_spatial_info = bool(planner_gets_spatial_info)
        self.full_observability = bool(full_observability)
        self.obs_range = int(mobile_agent_observation_range)
        self.starting_agent_coin = float(starting_agent_coin)
        assert self.starting_agent_coin >= 0.0
        self.isoelastic_eta = float(isoelastic_eta)
        assert 0.0 <= self.isoelastic_eta <= 1.0
        self.energy_cost = float(energy_cost)
        assert self.energy_cost >= 0
        self.energy_warmup_method = energy_warmup_method.lower()
        assert self.energy_warmup_method in ["decay", "auto"]
        self.energy_warmup_constant = float(energy_warmup_constant)
        assert self.energy_warmup_constant >= 0
        self.planner_reward_type = str(planner_reward_type).lower()
        if self.planner_reward_type not in _SWF:
            raise NotImplementedError("No valid planner reward selected!")
        self.mixing_weight_gini_vs_coin = float(mixing_weight_gini_vs_coin)
        assert 0 <= self.mixing_weight_gini_vs_coin <= 1.0

    # -- shared helpers ---------------------------------------------------------------------------
    def _place_randomly(self, rs, order, blocked):
        """Rejection-sample a free, accessible cell for each agent in `order`
        (layout_from_file.py:359-370 / dynamic_layout.py:418-429)."""
        H, W = self.env.world_size
        A = self.env.n_agents
        loc = -np.ones((A, 2), np.int16)
        taken = np.zeros((H, W), bool)
        for a in order:
            r, c = rs.randint(0, H), rs.randint(0, W)
            tries = 0
            while blocked[r, c] or taken[r, c]:
                r, c = rs.randint(0, H), rs.randint(0, W)
                tries += 1
                if tries > 200:
                    raise TimeoutError
            loc[a] = (r, c)
            taken[r, c] = True
        return loc

    def _component_resets(self, rs, st):
        """Component.reset() in component-list order (base_env.py:906-908)."""
        A = self.env.n_agents
        st["build_payment"], st["build_skill"], st["bonus_gather_prob"] = np.zeros(A), np.zeros(A), np.zeros(A)
        for comp in self.env.components:
            if comp.name == "Build":
                st["build_payment"], st["build_skill"] = comp.sample_skills(rs, A)
            elif comp.name == "Gather":
                st["bonus_gather_prob"] = comp.sample_skills(rs, A)

    def device_reset_tables(self):
        """Per-replica tables a device-side reset hands out again, besides the stream: {name: array [n_envs, ...]}."""
        return {}

    def scenario_spec_fields(self):
        return dict(
            obs_range=self.obs_range, planner_gets_spatial_info=int(self.planner_gets_spatial_info),
            full_observability=int(self.full_observability),
            isoelastic_eta=self.isoelastic_eta, energy_cost=self.energy_cost,
            energy_warmup_constant=self.energy_warmup_constant,
            energy_warmup_auto=int(self.energy_warmup_method == "auto"),
            planner_reward_type=_SWF[self.planner_reward_type],
            mixing_weight_gini_vs_coin=self.mixing_weight_gini_vs_coin)


scenario_registry = Registry(BaseScenario)


@scenario_registry.add
class LayoutFromFile(BaseScenario):
    name = "layout_from_file/simple_wood_and_stone"
    required_entities = ["Wood", "Stone", "Water"]

    def __init__(self, env, env_layout_file="quadrant_25x25_20each_30clump.txt", resource_regen_prob=0.01,
                 fixed_four_skill_and_loc=False, **kw):
        super().__init__(env, **kw)
        H, W = env.world_size
        path = os.path.join(MAP_DIR, env_layout_file)
        with open(path, "r") as f:
            self.env_layout_string = f.read()
        self.env_layout = self.env_layout_string.split(";")
        sym = {"W": "Wood", "S": "Stone", "@": "Water"}
        self.source_maps = {k: np.zeros((H, W), np.uint8) for k in sym.values()}
        for r, row in enumerate(self.env_layout):
            for c, ch in enumerate(row):
                if ch in sym:
                    self.source_maps[sym[ch]][r, c] = 1
        self.regen_weight = float(resource_regen_prob)
        assert 0 <= self.regen_weight <= 1
        self.fixed_four_skill_and_loc = bool(fixed_four_skill_and_loc)
        if self.fixed_four_skill_and_loc:
            self._init_fixed_four()

    def _init_fixed_four(self):
        """Average ranked Pareto skills + corner start cells (layout_from_file.py:165-247)."""
        env = self.env
        bm = env.get_component("Build")
        assert bm.skill_dist == "pareto"
        pmsm, A = bm.payment_max_skill_multiplier, env.n_agents
        H, W = env.world_size
        samples = np.random.RandomState(1).pareto(4, size=(100000, A))  # reference: np.random.seed(seed=1)
        ranked = np.sort(np.minimum(pmsm, (pmsm - 1) * samples + 1), axis=1).mean(axis=0)
        self._avg_ranked_skill = ranked * bm.payment
        corners = [(0, W - 1), (H - 1, 0), (0, 0), (W - 1, W - 1)]  # sic: the reference uses W for the last row
        groups = np.floor(np.arange(A) * (4 / A)).astype(int)
        count = np.zeros(4, int)
        self._ranked_locs = []
        for g in groups:
            k = count[g]
            dr, dc = k // 4, k % 4
            r0, c0 = corners[g]
            self._ranked_locs.append({0: (r0 + dr, c0 - dc), 1: (r0 - dr, c0 + dc),
                                      2: (r0 + dr, c0 + dc), 3: (r0 - dr, c0 - dc)}[int(g)])
            count[g] += 1

    def host_reset(self, rs, e=0):
        env = self.env
        A = env.n_agents
        st = dict(stone=self.source_maps["Stone"].copy(), wood=self.source_maps["Wood"].copy(),
                  stone_src=self.source_maps["Stone"].copy(), wood_src=self.source_maps["Wood"].copy(),
                  water=self.source_maps["Water"].copy())
        st["coin"] = np.full(A, self.starting_agent_coin)
        st["loc"] = self._place_randomly(rs, range(A), st["water"] > 0)
        self._component_resets(rs, st)
        if self.fixed_four_skill_and_loc:  # layout_from_file.py:580-586
            order = rs.permutation(A)
            for i, a in enumerate(order):
                r, c = self._ranked_locs[i]
                assert not st["water"][r, c], "fixed_four start cell is water"
                st["loc"][a] = (r, c)
                st["build_payment"][a] = self._avg_ranked_skill[i]
        return st

    def scenario_spec_fields(self):
        d = super().scenario_spec_fields()
        d.update(has_water=1, regen_weight=[self.regen_weight, self.regen_weight])
        # device-side reset with reference semantics (used by auto_reset)
        dists = {"none": 0, "pareto": 1, "lognormal": 2}
        comps = {c.name: c for c in self.env.components}
        b, g = comps.get("Build"), comps.get("Gather")
        ok = (b is None or b.skill_dist in dists) and (g is None or g.skill_dist in dists)
        d.update(reset_mode=1 if ok else 0,
                 build_skill_dist=dists.get(b.skill_dist, 0) if b else 0,
                 gather_skill_dist=dists.get(g.skill_dist, 0) if g else 0,
                 payment_max_skill_multiplier=b.payment_max_skill_multiplier if b else 1,
                 fixed_four=int(self.fixed_four_skill_and_loc),
                 ranked_locs=[list(map(int, rc)) for rc in getattr(self, "_ranked_locs", [])],
                 avg_ranked_skill=[float(v) for v in getattr(self, "_avg_ranked_skill", [])])
        return d


@scenario_registry.add
class Uniform(BaseScenario):
    name = "uniform/simple_wood_and_stone"
    required_entities = ["Wood", "Stone"]

    def __init__(self, env, starting_wood_coverage=0.025, wood_regen_halfwidth=0, wood_regen_weight=0.01,
                 wood_max_health=1, starting_stone_coverage=0.025, stone_regen_halfwidth=0, stone_regen_weight=0.01,
                 stone_max_health=1, wood_clumpiness=0.35, stone_clumpiness=0.5, gradient_steepness=8,
                 checker_source_blocks=False, **kw):
        super().__init__(env, **kw)
        H, W = env.world_size
        if starting_wood_coverage >= 1:
            starting_wood_coverage /= np.prod(env.world_size)
        if starting_stone_coverage >= 1:
            starting_stone_coverage /= np.prod(env.world_size)
        assert (starting_stone_coverage + starting_wood_coverage) < 0.5
        self.checker = bool(checker_source_blocks)
        cc, rr = np.meshgrid(np.arange(W) % 2, np.arange(H) % 2)
        self._checker_mask = (rr + cc) == 1
        m = 2 if self.checker else 1
        self.coverage = {"Wood": float(starting_wood_coverage) * m, "Stone": float(starting_stone_coverage) * m}
        assert 0 < self.coverage["Wood"] < 1 and 0 < self.coverage["Stone"] < 1
        self.regen_halfwidth = {"Wood": int(wood_regen_halfwidth), "Stone": int(stone_regen_halfwidth)}
        assert 0 <= self.regen_halfwidth["Wood"] <= 3 and 0 <= self.regen_halfwidth["Stone"] <= 3
        if int(wood_max_health) != 1 or int(stone_max_health) != 1:
            raise NotImplementedError("max_health != 1 is not on the GPU path")
        self.regen = {"Wood": float(wood_regen_weight), "Stone": float(stone_regen_weight)}
        assert 0 <= self.regen["Wood"] <= 1 and 0 <= self.regen["Stone"] <= 1
        self.clumpiness = {"Wood": float(wood_clumpiness), "Stone": float(stone_clumpiness)}
        assert all(0 <= v <= 1 for v in self.clumpiness.values())
        self.gradient_steepness = float(gradient_steepness)
        assert self.gradient_steepness >= 1.0
        self.source_prob_maps = self.make_source_prob_maps(self._ctor_stream())

    def _ctor_stream(self):
        """The stream the reference's constructor would draw from: the env's seeded stream when `seed=` was passed
        to make_env_instance (base_env.py:286-287 seeds before anything is built), else an unseeded one."""
        rs = self.env._rs
        return rs[0] if rs is not None else np.random.RandomState()

    def make_source_prob_maps(self, rs):
        """dynamic_layout.py:289-308"""
        H, W = self.env.world_size
        grad = np.arange(H)[:, None].repeat(W, axis=1) ** self.gradient_steepness
        grad = grad / np.mean(grad)
        # sic: both maps are scaled by the Wood coverage (dynamic_layout.py:302-306)
        return {"Wood": grad * self.coverage["Wood"], "Stone": grad[-1::-1] * self.coverage["Wood"]}

    def _generate_layout(self, rs):
        """Clumped random source placement, dynamic_layout.py:313-392 (same draws, same order)."""
        from scipy import signal

        H, W = self.env.world_size
        src = {}
        for _ in range(100):
            occupied = np.zeros((H, W), bool)
            src = {}
            for res in ("Wood", "Stone"):
                clump = 1 - np.clip(self.clumpiness[res], 0.0, 0.99)
                prob = self.source_prob_maps[res] * 0.1 * clump
                empty = ~occupied
                noise = rs.rand(H, W)
                cand = (noise < prob) * empty
                tries = 0
                while np.mean(cand) < self.coverage[res] * clump:
                    noise *= 0.9
                    cand = (noise < prob) * empty
                    tries += 1
                    if tries > 200:
                        break
                while np.mean(cand) < self.coverage[res]:
                    kernel = rs.randn(7, 7) > 0
                    grown = signal.convolve2d(cand + (0.2 * rs.randn(H, W)) - 0.25, kernel.astype(np.float32), "same")
                    cand = np.maximum(grown > 0, cand) * empty
                src[res] = cand
                occupied = occupied | (cand > 0)
            ok = True
            for res in ("Wood", "Stone"):
                q = np.mean(src[res]) / self.coverage[res]
                if not (1 / 1.4) <= q <= 1.4:
                    ok = False
            if ok:
                break
        if self.checker:
            src = {k: v * self._checker_mask for k, v in src.items()}
        return {k: (v > 0).astype(np.uint8) for k, v in src.items()}

    def _starting_layout(self, rs):
        """reset_starting_layout (dynamic_layout.py:313-392) -> (source maps, water map)."""
        H, W = self.env.world_size
        return self._generate_layout(rs), np.zeros((H, W), np.uint8)

    def host_reset(self, rs, e=0):
        A = self.env.n_agents
        src, water = self._starting_layout(rs)
        st = dict(stone=src["Stone"].copy(), wood=src["Wood"].copy(), stone_src=src["Stone"].copy(),
                  wood_src=src["Wood"].copy(), water=water)
        st["coin"] = np.full(A, self.starting_agent_coin)
        order = rs.permutation(A)  # world.get_random_order_agents()
        st["loc"] = self._place_randomly(rs, order, water > 0)
        self._component_resets(rs, st)
        return st

    dyn_layout_kind = 1   # aie_config.dyn_layout: the device-side twin of _generate_layout (0: none)

    def scenario_spec_fields(self):
        d = super().scenario_spec_fields()
        d.update(has_water=0, regen_weight=[self.regen["Stone"], self.regen["Wood"]],
                 regen_halfwidth=[self.regen_halfwidth["Stone"], self.regen_halfwidth["Wood"]])
        # device-side reset with reference semantics (auto_reset): clumped layout + random-order placement + skills
        dists = {"none": 0, "pareto": 1, "lognormal": 2}
        comps = {c.name: c for c in self.env.components}
        b, g = comps.get("Build"), comps.get("Gather")
        ok = self.dyn_layout_kind and (b is None or b.skill_dist in dists) and (g is None or g.skill_dist in dists)
        if ok:
            d.update(reset_mode=1, dyn_layout=int(self.dyn_layout_kind), dyn_checker=int(self.checker),
                     dyn_coverage=[self.coverage["Wood"], self.coverage["Stone"]],
                     dyn_clump=[float(1 - np.clip(self.clumpiness["Wood"], 0.0, 0.99)),
                                float(1 - np.clip(self.clumpiness["Stone"], 0.0, 0.99))],
                     dyn_prob=(None if self.dyn_layout_kind == 3 else
                               [np.asarray(self.source_prob_maps["Wood"], np.float64).tolist(),
                                np.asarray(self.source_prob_maps["Stone"], np.float64).tolist()]),
                     build_skill_dist=dists.get(b.skill_dist, 0) if b else 0,
                     gather_skill_dist=dists.get(g.skill_dist, 0) if g else 0,
                     payment_max_skill_multiplier=b.payment_max_skill_multiplier if b else 1)
        return d


@scenario_registry.add
class MultiZone(Uniform):
    """Wood / stone / mixed source zones on a shuffled partition grid (dynamic_layout.py:706-873).  The zone
    assignment is re-shuffled from the env's stream at every reset, before the clumped layout is drawn."""
    name = "multi_zone/simple_wood_and_stone"
    dyn_layout_kind = 3   # the zone assignment is re-shuffled on the device at every reset (np.random.shuffle), then the layout

    def __init__(self, env, num_partitions_row=8, num_partitions_col=8, num_wood_zones=6, num_stone_zones=6,
                 num_wood_and_stone_zones=4, **kw):
        self.num_partitions_row = num_partitions_row
        self.num_partitions_col = num_partitions_col
        self.zone_specs = {"Wood": (0, num_wood_zones), "Stone": (1, num_stone_zones),
                           "WoodStone": (2, num_wood_and_stone_zones)}
        super().__init__(env, **kw)
        if env._rs is not None:   # the constructor's shuffle advances every replica's seeded stream alike
            n_regions = self.num_partitions_row * self.num_partitions_col
            for rs in env._rs[1:]:
                rs.shuffle(np.arange(n_regions))

    def scenario_spec_fields(self):
        d = super().scenario_spec_fields()
        if d.get("dyn_layout") == 3:
            assert self.num_partitions_row * self.num_partitions_col <= 128, "device-side MultiZone reset: at most 128 regions"
            d.update(mz_partitions=[int(self.num_partitions_row), int(self.num_partitions_col)],
                     mz_zones=[int(self.zone_specs[k][1]) for k in ("Wood", "Stone", "WoodStone")])
            d.pop("dyn_prob", None)
        return d

    def make_source_prob_maps(self, rs):
        """dynamic_layout.py:778-864 (one np.random.shuffle of the region -> zone-type vector)."""
        H, W = self.env.world_size
        idx = [v[0] for v in self.zone_specs.values()]
        per_type = [v[1] for v in self.zone_specs.values()]
        n_zones = sum(per_type)
        n_regions = self.num_partitions_row * self.num_partitions_col
        assert n_regions >= n_zones
        size_r = int(np.ceil(H / self.num_partitions_row))
        size_c = int(np.ceil(W / self.num_partitions_col))
        grid = np.concatenate([np.repeat(idx, per_type), np.array([-1] * (n_regions - n_zones))])
        rs.shuffle(grid)
        grid = grid.reshape((self.num_partitions_row, self.num_partitions_col))
        out = {}
        for res, own in (("Wood", 0), ("Stone", 1)):
            prob = np.where((grid == own) | (grid == 2), np.ones_like(grid), np.zeros_like(grid))
            prob = np.kron(prob, np.ones((size_r, size_c)))[:H, :W]
            assert prob.shape == (H, W), "World not correct size!"
            out[res] = prob / np.mean(prob)
        # sic: both maps are scaled by the Wood coverage (dynamic_layout.py:860-863)
        return {"Wood": out["Wood"] * self.coverage["Wood"], "Stone": out["Stone"] * self.coverage["Wood"]}

    def _starting_layout(self, rs):
        self.source_prob_maps = self.make_source_prob_maps(rs)  # dynamic_layout.py:866-872
        return super()._starting_layout(rs)


@scenario_registry.add
class Quadrant(Uniform):
    """Two water lines with gaps split the world into four quadrants; wood concentrates towards the bottom rows,
    stone towards the left columns (dynamic_layout.py:876-1021)."""
    name = "quadrant/simple_wood_and_stone"
    required_entities = Uniform.required_entities + ["Water"]
    dyn_layout_kind = 2

    def __init__(self, env, **kw):
        super().__init__(env, **kw)
        H, W = env.world_size
        o0, o1 = 0.2, 0.35
        rn = (0.5 + np.arange(H)) / H
        cn = (0.5 + np.arange(W)) / W
        rseg = ((rn < o0) + (rn > o1)) * ((rn < 1 - o1) + (rn > 1 - o0))
        cseg = ((cn < o0) + (cn > o1)) * ((cn < 1 - o1) + (cn > 1 - o0))
        water = np.zeros((H, W))
        water[:, H // 2] = rseg     # sic: the reference indexes the column with height // 2 ...
        water[W // 2, :] = cseg     # ... and the row with width // 2 (dynamic_layout.py:951-952)
        self._water = water
        for k, v in self.source_prob_maps.items():
            v = v * (1 - self._water)
            self.source_prob_maps[k] = v / np.sum(v)

    def make_source_prob_maps(self, rs):
        """dynamic_layout.py:960-990"""
        H, W = self.env.world_size
        g = np.arange(H)[:, None].repeat(W, axis=1) ** (self.gradient_steepness / 2)
        w_grad = g[::-1]
        g = np.arange(W)[None].repeat(H, axis=0) ** (self.gradient_steepness / 2)
        s_grad = g[:, ::-1]
        tot = s_grad + w_grad
        s_grad, w_grad = tot * s_grad, tot * w_grad
        return {"Stone": s_grad / np.sum(s_grad), "Wood": w_grad / np.sum(w_grad)}

    def _starting_layout(self, rs):
        """dynamic_layout.py:992-1021: the uniform layout, nothing on the water lines, then the water."""
        H, W = self.env.world_size
        src, _ = super()._starting_layout(rs)
        for k in src:
            src[k][:, H // 2] = 0
            src[k][W // 2, :] = 0
        return src, (self._water > 0).astype(np.uint8)

    def scenario_spec_fields(self):
        d = super().scenario_spec_fields()
        d.update(has_water=1)
        return d


@scenario_registry.add
class SplitLayout(LayoutFromFile):
    """layout_from_file with a water row through the middle, rank-averaged Pareto build skills handed out in a random
    order, and the agents of the chosen skill ranks placed above the water (layout_from_file.py:654-800)."""
    name = "split_layout/simple_wood_and_stone"

    def __init__(self, env, water_row=None, skill_rank_of_top_agents=None, **kw):
        super().__init__(env, **kw)
        if self.fixed_four_skill_and_loc:
            raise ValueError("The split layout scenario does not support fixed_four_skill_and_loc. "
                             "Set this to False.")
        H, W = env.world_size
        if water_row is None:
            self._water_line = H // 2
        else:
            self._water_line = int(water_row)
            assert 0 < self._water_line < H - 1
        for k, m in self.source_maps.items():
            m[self._water_line, :] = 1 if k == "Water" else 0
        if skill_rank_of_top_agents is None:
            skill_rank_of_top_agents = [0]
        if isinstance(skill_rank_of_top_agents, (int, float)):
            self.skill_rank_of_top_agents = [int(skill_rank_of_top_agents)]
        elif isinstance(skill_rank_of_top_agents, (tuple, list)):
            self.skill_rank_of_top_agents = list(set(skill_rank_of_top_agents))
        else:
            raise TypeError("skill_rank_of_top_agents must be a scalar index, or a list of scalar indices.")
        for rank in self.skill_rank_of_top_agents:
            assert 0 <= rank < env.n_agents
        assert 0 < len(self.skill_rank_of_top_agents) < env.n_agents
        bm = env.get_component("Build")
        assert bm.skill_dist == "pareto"
        # The reference draws its 100000 x n_agents Pareto table from the global stream inside the constructor
        # (layout_from_file.py:747); here every replica draws its own table from its own stream, at construction
        # when `seed=` was passed (as base_env.py:286-287 seeds first), else from an unseeded stream.
        pmsm, A = bm.payment_max_skill_multiplier, env.n_agents
        self._split_ranked_skill = np.zeros((env.n_envs, A))
        for e in range(env.n_envs):
            rs = env._rs[e] if env._rs is not None else np.random.RandomState()
            samples = rs.pareto(4, size=(100000, A))
            ranked = np.sort(np.minimum(pmsm, (pmsm - 1) * samples + 1), axis=1).mean(axis=0)
            self._split_ranked_skill[e] = (ranked * bm.payment)[::-1]

    def host_reset(self, rs, e=0):
        st = super().host_reset(rs, e)
        env = self.env
        A = env.n_agents
        H, W = env.world_size
        # additional_reset_steps (layout_from_file.py:766-790): everybody is taken off the map and re-placed
        order = rs.permutation(A)
        loc = -np.ones((A, 2), np.int16)
        taken = np.zeros((H, W), bool)
        blocked = st["water"] > 0
        for i, a in enumerate(order):
            st["build_payment"][a] = self._split_ranked_skill[e, i]
            r_min, r_max = (0, self._water_line) if i in self.skill_rank_of_top_agents else (self._water_line + 1, H)
            r, c = rs.randint(r_min, r_max), rs.randint(0, W)
            tries = 0
            while blocked[r, c] or taken[r, c]:
                r, c = rs.randint(r_min, r_max), rs.randint(0, W)
                tries += 1
                if tries > 200:
                    raise TimeoutError
            loc[a] = (r, c)
            taken[r, c] = True
        st["loc"] = loc
        st["split_skill"] = self._split_ranked_skill[e].copy()   # the device-side reset hands these out again
        return st

    def device_reset_tables(self):
        return {"split_skill": self._split_ranked_skill}

    def scenario_spec_fields(self):
        d = super().scenario_spec_fields()   # reset_mode 1 when the skill distributions have a device-side sampler
        top = 0
        for rank in self.skill_rank_of_top_agents:
            top |= 1 << int(rank)
        d.update(split_layout=1, split_water_row=int(self._water_line), split_top_ranks=top)
        return d


@scenario_registry.add
class OneStepEconomy(BaseScenario):
    """reference: scenarios/one_step_economy/one_step_economy.py:15-336.  Two-step episodes: the planner sets taxes, then
    every agent picks its hours of labor.  No map, no spatial observations; utilities are coin minus a labor cost.
    Its reset draws nothing, so the device's snapshot restore IS the reference's reset."""
    name = "one-step-economy"
    agent_subclasses = ["BasicMobileAgent", "BasicPlanner"]
    required_entities = ["Coin"]

    def __init__(self, env, agent_reward_type="coin_minus_labor_cost", isoelastic_eta=0.23, labor_exponent=2.0,
                 labor_cost=1.0, planner_reward_type="inv_income_weighted_utility", mixing_weight_gini_vs_coin=0):
        self.env = env
        self.agent_reward_type = str(agent_reward_type)
        if self.agent_reward_type not in ("isoelastic_coin_minus_labor", "coin_minus_labor_cost"):
            raise NotImplementedError("unknown agent_reward_type")
        self.isoelastic_eta = float(isoelastic_eta)
        self.labor_exponent = float(labor_exponent)
        self.labor_cost = float(labor_cost)
        self.planner_reward_type = str(planner_reward_type)
        if self.planner_reward_type not in ("coin_eq_times_productivity", "inv_income_weighted_utility"):
            print("No valid planner reward selected!")
            raise NotImplementedError
        self.mixing_weight_gini_vs_coin = float(mixing_weight_gini_vs_coin)
        if self.agent_reward_type == "isoelastic_coin_minus_labor":
            assert 0.0 <= self.isoelastic_eta <= 1.0
        else:
            assert self.labor_exponent > 1.0
        labor = env._components_dict.get("SimpleLabor")
        if labor is None or any(c.name not in ("SimpleLabor", "PeriodicBracketTax") for c in env._components):
            raise NotImplementedError("the one-step-economy runs with SimpleLabor (+ PeriodicBracketTax)")
        # the reference's component constructors run after the seeding and before the scenario's: SimpleLabor's skill table
        # is the only constructor-time draw
        streams = env._rs if env._rs is not None else [np.random.RandomState() for _ in range(env.n_envs)]
        labor.draw_skills(streams)

    def host_reset(self, rs, e=0):
        """reset_agent_states + component resets (one_step_economy.py:93-109, simple_labor.py:88-91): nothing is drawn."""
        env = self.env
        A = env.n_agents
        H, W = env.world_size
        z = np.zeros((H, W), np.uint8)
        skills = env._components_dict["SimpleLabor"].skills[e]
        return dict(stone=z, wood=z.copy(), stone_src=z.copy(), wood_src=z.copy(), water=z.copy(),
                    loc=np.zeros((A, 2), np.int16),   # nobody is placed (one_step_economy.py:93-105); not observed
                    coin=np.zeros(A), inv_stone=np.zeros(A, np.int32),
                    inv_wood=np.zeros(A, np.int32),
                    build_payment=np.zeros(A),              # record reuse: cumulative production
                    build_skill=np.asarray(skills, float),  # record reuse: the SimpleLabor skill
                    bonus_gather_prob=np.zeros(A))

    def scenario_spec_fields(self):
        return dict(scenario_kind=1, has_water=0, obs_range=0, planner_gets_spatial_info=0, regen_weight=[0.0, 0.0],
                    isoelastic_eta=self.isoelastic_eta, energy_cost=0.0, energy_warmup_constant=0.0, energy_warmup_auto=0,
                    planner_reward_type=_SWF[self.planner_reward_type],
                    mixing_weight_gini_vs_coin=self.mixing_weight_gini_vs_coin,
                    agent_reward_type=int(self.agent_reward_type == "coin_minus_labor_cost"),
                    labor_exponent=self.labor_exponent, labor_cost=self.labor_cost, reset_mode=0)
