// aie_host.h — host-side logic of the C-ABI that needs no CUDA: config validation, record layout,
// observation/mask "programs" (the reference's sorted-key flattening resolved once), packing a host reset
// snapshot into state records and unpacking a record for test readback.
#pragma once
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/aie_b200.h"
#include "aie_layout.h"

namespace aie {

inline int align16(int x) { return (x + 15) & ~15; }
inline uint64_t host_mix64(uint64_t x) {  // splitmix64 finaliser (same function as mix64 in aie_core.cuh)
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

struct FlatKey { std::string key; int kind, payload, n; };  // payload of element i = payload + i

// Mirrors BaseEnvironment._build_packager / _package (base_env.py:562-612): every scalar / 1-D field is
// concatenated in sorted key order.  Keys are the reference's: "<Component>-<obs>" / "world-<obs>" / "time".
inline int build_prog(std::vector<FlatKey> keys, uint16_t *prog, int cap, std::vector<aie_flat_field> *layout = nullptr) {
    std::sort(keys.begin(), keys.end(), [](const FlatKey &a, const FlatKey &b) { return a.key < b.key; });
    int n = 0;
    for (const FlatKey &k : keys) {
        if (layout) {  // where this field sits in the flat vector (aie_get_flat_layout)
            aie_flat_field f;
            memset(&f, 0, sizeof(f));
            snprintf(f.key, sizeof(f.key), "%s", k.key.c_str());
            f.offset = n; f.size = k.n;
            layout->push_back(f);
        }
        for (int i = 0; i < k.n; i++) {
            if (n >= cap) return -1;
            prog[n++] = AIE_FLAT_ENTRY(k.kind, k.payload + i);
        }
    }
    return n;
}

// Returns 0 or AIE_EINVAL with a message in err.
inline int build_devcfg(const aie_config &u, int n_envs, DevCfg &c, Tables &tb, std::string &err,
                        std::vector<aie_flat_field> *layouts = nullptr /* [3]: agent flat, planner flat, p<i> */) {
    memset(&c, 0, sizeof(c));
    memset(&tb, 0, sizeof(tb));
    auto bad = [&](const char *m) { err = m; return AIE_EINVAL; };
    if (u.abi_version != AIE_ABI_VERSION) return bad("abi_version mismatch");
    if (u.obs_dtype != AIE_OBS_F32 && u.obs_dtype != AIE_OBS_BF16) return bad("obs_dtype must be AIE_OBS_F32 or AIE_OBS_BF16");
    if (n_envs < 1) return bad("n_envs must be >= 1");
    if (u.n_agents < 2 || u.n_agents > AIE_MAX_AGENTS) return bad("n_agents must be in [2, 64]");
    if (u.height < 1 || u.width < 1 || u.height > 256 || u.width > 256) return bad("world size must be within 256x256");
    if (u.episode_length < 1 || u.episode_length >= (1 << 23)) return bad("episode_length out of range");
    if (u.n_components < 1 || u.n_components > AIE_MAX_COMPONENTS) return bad("1..8 components");
    if (u.obs_range < 0 || u.obs_range > 32) return bad("mobile_agent_observation_range out of range");
    c.A = u.n_agents; c.H = u.height; c.W = u.width; c.HW = u.height * u.width; c.T = u.episode_length;
    c.multi_action = u.multi_action_agents ? 1 : 0;
    c.n_comp = u.n_components;
    for (int i = 0; i < u.n_components; i++) {
        int k = u.components[i];
        if (k < 0 || k >= COMP_KINDS) return bad("unknown component kind");
        if (c.has[k]) return bad("duplicate component");
        c.comp[i] = k; c.has[k] = 1;
    }
    c.one_step = u.scenario_kind == 1 ? 1 : 0;
    if (u.scenario_kind != 0 && u.scenario_kind != 1) return bad("unknown scenario_kind");
    if (c.one_step) {   // one_step_economy.py: SimpleLabor (+ PeriodicBracketTax), nothing spatial
        for (int i = 0; i < c.n_comp; i++)
            if (c.comp[i] != COMP_LABOR && c.comp[i] != COMP_TAX) return bad("one-step-economy takes SimpleLabor and PeriodicBracketTax only");
        if (!c.has[COMP_LABOR]) return bad("one-step-economy needs the SimpleLabor component");
        if (u.agent_reward_type != 0 && u.agent_reward_type != 1) return bad("unknown agent_reward_type");
        if (u.agent_reward_type == 1 && !(u.labor_exponent > 1.0)) return bad("labor_exponent must be > 1");
        if (!(u.labor_skill_scale > 0.0)) return bad("labor_skill_scale (payment_max_skill_multiplier) must be > 0");
        if (u.planner_reward_type == 1) return bad("one-step-economy has no inv_income_weighted_coin_endowments planner reward");
        if (u.reset_mode != 0) return bad("one-step-economy resets from the snapshot (its reset draws nothing)");
        if (u.full_observability || u.planner_gets_spatial_info) return bad("one-step-economy has no spatial observations");
    } else if (c.has[COMP_LABOR]) return bad("SimpleLabor belongs to the one-step-economy scenario");
    c.no_spatial = c.one_step;
    c.agent_reward_type = u.agent_reward_type; c.labor_exponent = u.labor_exponent; c.labor_cost = u.labor_cost;
    c.labor_mask_first = u.labor_mask_first_step ? 1 : 0; c.labor_skill_scale = u.labor_skill_scale;
    c.has_water = u.has_water ? 1 : 0;
    c.M = c.has_water ? 6 : 5;
    c.w = u.obs_range; c.win = 2 * u.obs_range + 1;
    c.planner_spatial = u.planner_gets_spatial_info ? 1 : 0;
    c.obs_scaling = u.allow_observation_scaling ? 1 : 0;
    for (int r = 0; r < 2; r++) {
        double w = u.regen_weight[r];
        if (!(w >= 0.0 && w <= 1.0)) return bad("regen weight must be in [0, 1]");
        c.regen_thresh[r] = (uint64_t)ceil(ldexp(w, 53));  // exact: N / 2^53 < w  <=>  N < ceil(w * 2^53)
        const int hw = u.regen_halfwidth[r];
        if (hw < 0 || hw > 3) return bad("regen_halfwidth must be in [0, 3]");
        c.regen_hw[r] = hw;
        // scipy.signal.convolve2d accumulates health * kernel terms in float64; every kernel entry is
        // (regen_weight * 1.0) / d^2 and health is 0/1, so the value at a cell is n sequential additions of that entry
        const int d = 1 + 2 * hw;
        const double kv = (w * 1.0) / (double)(d * d);
        double p = 0.0;
        for (int n = 0; n < 50; n++) {
            c.regen_tab[r][n] = p >= 1.0 ? (1ull << 53) : (uint64_t)ceil(ldexp(p, 53));
            p += kv;
        }
    }
    c.eta = u.isoelastic_eta; c.energy_cost = u.energy_cost; c.warm_const = u.energy_warmup_constant;
    if (!(c.eta >= 0.0 && c.eta <= 1.0)) return bad("isoelastic_eta must be in [0, 1]");
    c.warm_auto = u.energy_warmup_auto ? 1 : 0;
    c.swf = u.planner_reward_type;
    if (c.swf < 0 || c.swf > 2) return bad("unknown planner_reward_type");
    c.mix = u.mixing_weight_gini_vs_coin;
    c.build_payment = u.build_payment; c.build_labor = u.build_labor;
    c.move_labor = u.move_labor; c.collect_labor = u.collect_labor; c.order_labor = u.order_labor;
    c.P = u.max_bid_ask + 1; c.D = u.order_duration; c.K = u.max_num_orders;
    if (c.has[COMP_CDA]) {
        if (c.P < 2 || c.P > AIE_MAX_PRICE_LEVELS) return bad("max_bid_ask must be in [1, 31]");
        if (c.D < 1 || c.D > 4095) return bad("order_duration must be in [1, 4095]");
        if (c.K < 1 || c.K > 255) return bad("max_num_orders must be in [1, 255]");
    } else { c.P = 1; c.D = 1; c.K = 1; }
    c.K_magic = c.K == 1 ? 0u : (uint32_t)((1ull << 32) / (uint64_t)c.K) + 1u;
    c.tax_model = u.tax_model; c.disable_taxes = u.disable_taxes ? 1 : 0; c.period = u.period;
    c.B = u.n_brackets; c.R = u.n_disc_rates;
    if (c.has[COMP_TAX]) {
        if (c.tax_model != AIE_TAX_MODEL_WRAPPER && c.tax_model != AIE_TAX_FIXED_RATES && c.tax_model != AIE_TAX_SAEZ)
            return bad("unsupported tax_model");
        if (c.B < 2 || c.B > AIE_MAX_BRACKETS) return bad("n_brackets must be in [2, 16]");
        if (c.tax_model == AIE_TAX_MODEL_WRAPPER && (c.R < 1 || c.R > AIE_MAX_RATES)) return bad("n_disc_rates must be in [1, 64]");
        if (c.period < 1) return bad("tax period must be >= 1");
        for (int b = 0; b < c.B; b++) { c.cutoffs[b] = u.bracket_cutoffs[b]; c.fixed_rates[b] = u.fixed_rates[b]; }
        for (int r = 0; r < c.R; r++) { c.disc_rates[r] = u.disc_rates[r]; c.ann_full = fmax(c.ann_full, fabs(u.disc_rates[r])); }
    } else { c.B = 0; c.R = 0; c.period = 1; }
    c.tax_annealing = u.tax_annealing ? 1 : 0;
    c.ann_warm = u.annealing_warmup; c.ann_slope = u.annealing_slope; c.rate_max = u.rate_max; c.rate_min = u.rate_min;
    c.auto_reset = u.auto_reset ? 1 : 0;
    c.reset_mode = u.reset_mode;
    if (c.reset_mode != 0 && c.reset_mode != 1) return bad("unknown reset_mode");
    c.build_skill_dist = u.build_skill_dist; c.gather_skill_dist = u.gather_skill_dist;
    if (c.build_skill_dist < 0 || c.build_skill_dist > 2 || c.gather_skill_dist < 0 || c.gather_skill_dist > 2)
        return bad("device-side reset supports skill_dist 'none', 'pareto' and 'lognormal'");
    c.pmsm = u.payment_max_skill_multiplier; c.fixed_four = u.fixed_four ? 1 : 0;
    for (int i = 0; i < c.A; i++) {
        c.ranked_locs[i][0] = u.ranked_locs[i][0]; c.ranked_locs[i][1] = u.ranked_locs[i][1];
        c.avg_ranked_skill[i] = u.avg_ranked_skill[i];
        if (c.reset_mode == 1 && c.fixed_four &&
            (c.ranked_locs[i][0] < 0 || c.ranked_locs[i][0] >= c.H || c.ranked_locs[i][1] < 0 || c.ranked_locs[i][1] >= c.W))
            return bad("fixed_four start cell outside the world");
    }
    c.n_envs = n_envs;
    c.obs_bf16 = u.obs_dtype == AIE_OBS_BF16 ? 1 : 0;

    // action subspaces in component-list order (base_agent.py:124-169)
    int lo = 1, n_single = 0;
    for (int i = 0; i < c.n_comp; i++) {
        auto add = [&](int kind, int cc, int n) {
            c.sub_kind[c.n_sub] = kind; c.sub_c[c.n_sub] = cc; c.sub_n[c.n_sub] = n; c.sub_lo[c.n_sub] = lo;
            lo += n; n_single += n; c.n_sub++;
        };
        if (c.comp[i] == COMP_BUILD) add(SUB_BUILD, 0, 1);
        else if (c.comp[i] == COMP_CDA) { for (int cc = 0; cc < 2; cc++) { add(SUB_BUY, cc, c.P); add(SUB_SELL, cc, c.P); } }
        else if (c.comp[i] == COMP_GATHER) add(SUB_GATHER, 0, 4);
        else if (c.comp[i] == COMP_LABOR) add(SUB_LABOR, 0, 100);   // simple_labor.py:56 num_labor_hours
    }
    c.n_act_a = c.multi_action ? c.n_sub : 1;
    if (c.n_sub == 0) return bad("mobile agents need at least one action component");
    c.planner_acts = (c.has[COMP_TAX] && c.tax_model == AIE_TAX_MODEL_WRAPPER && !c.disable_taxes) ? 1 : 0;
    c.planner_single = (c.planner_acts && u.single_action_planner) ? 1 : 0;
    c.full_obs = u.full_observability ? 1 : 0;
    c.a_map_elems = c.no_spatial ? 0 : (c.full_obs ? c.M * c.HW : (c.M + 1) * c.win * c.win);
    c.a_idx_elems = c.no_spatial ? 0 : (c.full_obs ? 2 * c.HW : 2 * c.win * c.win);
    c.split_layout = (u.split_layout && c.reset_mode == 1) ? 1 : 0;
    c.split_water_row = u.split_water_row; c.split_top_ranks = u.split_top_ranks;
    if (c.split_layout && (c.split_water_row < 1 || c.split_water_row >= c.H - 1)) return bad("split_water_row outside the world");
    if (c.split_layout && c.fixed_four) return bad("split_layout does not support fixed_four_skill_and_loc");
    c.dyn_layout = (c.reset_mode == 1) ? u.dyn_layout : 0;
    if (c.dyn_layout < 0 || c.dyn_layout > 3) return bad("unknown dyn_layout");
    if ((c.dyn_layout == 1 || c.dyn_layout == 2) && !u.dyn_prob) return bad("dyn_layout needs the source probability maps (dyn_prob)");
    if (c.dyn_layout == 3) {
        c.mz_rows = u.mz_partitions[0]; c.mz_cols = u.mz_partitions[1];
        if (c.mz_rows < 1 || c.mz_cols < 1 || c.mz_rows * c.mz_cols > 128) return bad("MultiZone: 1..128 regions");
        int total = 0;
        for (int i = 0; i < 3; i++) { c.mz_zones[i] = u.mz_zones[i]; if (c.mz_zones[i] < 0) return bad("MultiZone: negative zone count"); total += c.mz_zones[i]; }
        if (total > c.mz_rows * c.mz_cols) return bad("MultiZone: more zones than regions");
        c.mz_psr = (c.H + c.mz_rows - 1) / c.mz_rows; c.mz_psc = (c.W + c.mz_cols - 1) / c.mz_cols;   // int(np.ceil(size / partitions))
    }
    if (c.dyn_layout && c.fixed_four) return bad("dynamic layouts have no fixed_four_skill_and_loc");
    c.dyn_checker = u.dyn_checker ? 1 : 0;
    for (int i = 0; i < 2; i++) {
        c.dyn_cov[i] = u.dyn_coverage[i]; c.dyn_clump[i] = u.dyn_clump[i];
        if (c.dyn_layout && !(c.dyn_cov[i] > 0.0 && c.dyn_cov[i] < 1.0 && c.dyn_clump[i] > 0.0 && c.dyn_clump[i] <= 1.0))
            return bad("dyn_coverage must be in (0, 1) and dyn_clump in (0, 1]");
    }
    c.ext = (c.planner_single || c.regen_hw[0] || c.regen_hw[1] || c.full_obs || c.split_layout || c.one_step ||
             (c.has[COMP_TAX] && (c.tax_model == AIE_TAX_FIXED_RATES || c.tax_model == AIE_TAX_SAEZ) && u.tax_annealing) ||
             (c.reset_mode == 1 && (c.build_skill_dist == 2 || c.gather_skill_dist == 2))) ? 1 : 0;
    c.n_act_p = c.planner_acts ? (c.planner_single ? 1 : c.B) : 0;
    c.Na = c.multi_action ? n_single + c.n_sub : 1 + n_single;
    c.Np = c.planner_acts ? (c.planner_single ? 1 + c.B * c.R : c.B * (1 + c.R)) : 1;
    if (c.Na > MAX_MASK) return bad("agent action mask too long");
    if (c.planner_single && c.Np > MAX_MASK) return bad("single-action planner mask too long (1 + n_brackets * n_disc_rates > 160)");

    c.sh_curr_rates = SH_PRICE_HIST + 2 * c.P;
    c.sh_last_incomes = c.sh_curr_rates + 16;
    c.sh_full = c.sh_last_incomes + c.A;  // full bid / ask counts [side][commodity][P]
    c.sh_count = c.sh_full + 4 * c.P;
    uint16_t mask_prog[MAX_MASK], prog_a[MAX_FLAT], prog_p[MAX_FLAT], prog_pa[16];
    // mask program (base_agent.py:440-460)
    {
        uint16_t *mp = mask_prog;
        int n = 0;
        if (!c.multi_action) mp[n++] = AIE_MASK_ENTRY(MS_ONE, 0);
        for (int si = 0; si < c.n_sub; si++) {
            if (c.multi_action) mp[n++] = AIE_MASK_ENTRY(MS_ONE, 0);
            for (int j = 0; j < c.sub_n[si]; j++) {
                if (c.sub_kind[si] == SUB_BUILD) mp[n++] = AIE_MASK_ENTRY(MS_BUILD, 0);
                else if (c.sub_kind[si] == SUB_BUY) mp[n++] = AIE_MASK_ENTRY(MS_BUY0 + c.sub_c[si], j);
                else if (c.sub_kind[si] == SUB_SELL) mp[n++] = AIE_MASK_ENTRY(MS_SELL0 + c.sub_c[si], j);
                else if (c.sub_kind[si] == SUB_LABOR) mp[n++] = AIE_MASK_ENTRY(MS_LABOR, j);
                else mp[n++] = AIE_MASK_ENTRY(MS_G0 + j, 0);
            }
        }
    }
    // flat programs: every scalar / 1-D observation field, concatenated in sorted key order
    {
        static const char *CN[2] = {"Stone", "Wood"};
        std::vector<FlatKey> ka, kp, kpa;
        auto K = [](const std::string &k, int kind, int payload, int n) { return FlatKey{k, kind, payload, n}; };
        if (c.one_step) {   // one_step_economy.py:138-160: nothing for the agents, two scalars for the planner
            ka.push_back(K("time", FK_SHARED, SH_TIME, 1)); kp.push_back(K("time", FK_SHARED, SH_TIME, 1));
            kp.push_back(K("world-normalized_per_capita_productivity", FK_SHARED, SH_ONE_PROD, 1));
            kp.push_back(K("world-equality", FK_SHARED, SH_ONE_EQ, 1));
            ka.push_back(K("SimpleLabor-skill", FK_AGENT, AS_LABOR_SKILL, 1));   // simple_labor.py:128-134
        } else {
        if (!c.full_obs) { ka.push_back(K("world-loc-row", FK_AGENT, AS_LOC_ROW, 1)); ka.push_back(K("world-loc-col", FK_AGENT, AS_LOC_COL, 1)); }
        ka.push_back(K("world-inventory-Coin", FK_AGENT, AS_INV_COIN, 1)); ka.push_back(K("world-inventory-Stone", FK_AGENT, AS_INV_STONE, 1));
        ka.push_back(K("world-inventory-Wood", FK_AGENT, AS_INV_WOOD, 1)); ka.push_back(K("time", FK_SHARED, SH_TIME, 1));
        kp.push_back(K("world-inventory-Coin", FK_SHARED, SH_ZERO, 1)); kp.push_back(K("world-inventory-Stone", FK_SHARED, SH_ZERO, 1));
        kp.push_back(K("world-inventory-Wood", FK_SHARED, SH_ZERO, 1)); kp.push_back(K("time", FK_SHARED, SH_TIME, 1));
        }
        // with full_observability the scenario sets no p<i> entries at all (layout_from_file.py:465-472 vs :509-513)
        if (!c.full_obs && !c.one_step) {
            kpa.push_back(K("world-inventory-Coin", FK_AGENT, AS_INV_COIN, 1)); kpa.push_back(K("world-inventory-Stone", FK_AGENT, AS_INV_STONE, 1));
            kpa.push_back(K("world-inventory-Wood", FK_AGENT, AS_INV_WOOD, 1));
        }
        if (c.planner_spatial && !c.full_obs) { kpa.push_back(K("world-loc-row", FK_AGENT, AS_LOC_ROW, 1)); kpa.push_back(K("world-loc-col", FK_AGENT, AS_LOC_COL, 1)); }
        if (c.has[COMP_BUILD]) { ka.push_back(K("Build-build_payment", FK_AGENT, AS_BUILD_PAYMENT, 1)); ka.push_back(K("Build-build_skill", FK_AGENT, AS_BUILD_SKILL, 1)); }
        if (c.has[COMP_GATHER]) ka.push_back(K("Gather-bonus_gather_prob", FK_AGENT, AS_BONUS, 1));
        if (c.has[COMP_CDA])
            for (int cc = 0; cc < 2; cc++) {
                std::string s = std::string("ContinuousDoubleAuction-"), r = std::string("-") + CN[cc];
                ka.push_back(K(s + "market_rate" + r, FK_SHARED, SH_MARKET_RATE + cc, 1));
                ka.push_back(K(s + "price_history" + r, FK_SHARED, SH_PRICE_HIST + cc * c.P, c.P));
                ka.push_back(K(s + "available_asks" + r, FK_AVAIL, (2 + cc) * c.P, c.P));
                ka.push_back(K(s + "available_bids" + r, FK_AVAIL, cc * c.P, c.P));
                ka.push_back(K(s + "my_asks" + r, FK_MY, (2 + cc) * c.P, c.P));
                ka.push_back(K(s + "my_bids" + r, FK_MY, cc * c.P, c.P));
                kp.push_back(K(s + "market_rate" + r, FK_SHARED, SH_MARKET_RATE + cc, 1));
                kp.push_back(K(s + "price_history" + r, FK_SHARED, SH_PRICE_HIST + cc * c.P, c.P));
                kp.push_back(K(s + "full_asks" + r, FK_SHARED, c.sh_full + (2 + cc) * c.P, c.P));
                kp.push_back(K(s + "full_bids" + r, FK_SHARED, c.sh_full + cc * c.P, c.P));
            }
        if (c.has[COMP_TAX]) {
            std::string s = "PeriodicBracketTax-";
            for (std::vector<FlatKey> *v : {&ka, &kp}) {
                v->push_back(K(s + "is_tax_day", FK_SHARED, SH_TAX_IS_TAX_DAY, 1)); v->push_back(K(s + "is_first_day", FK_SHARED, SH_TAX_IS_FIRST, 1));
                v->push_back(K(s + "tax_phase", FK_SHARED, SH_TAX_PHASE, 1)); v->push_back(K(s + "last_incomes", FK_SHARED, c.sh_last_incomes, c.A));
                v->push_back(K(s + "curr_rates", FK_SHARED, c.sh_curr_rates, c.B));
            }
            ka.push_back(K(s + "marginal_rate", FK_AGENT, AS_TAX_MARG, 1));
            kpa.push_back(K(s + "last_income", FK_AGENT, AS_TAX_LAST_INCOME, 1)); kpa.push_back(K(s + "last_marginal_rate", FK_AGENT, AS_TAX_LAST_MARG, 1));
            kpa.push_back(K(s + "curr_marginal_rate", FK_AGENT, AS_TAX_MARG, 1));
        }
        c.Fa = build_prog(ka, prog_a, MAX_FLAT, layouts ? &layouts[0] : nullptr);
        c.Fp = build_prog(kp, prog_p, MAX_FLAT, layouts ? &layouts[1] : nullptr);
        c.Fpa = build_prog(kpa, prog_pa, 16, layouts ? &layouts[2] : nullptr);
        if (c.Fa < 0 || c.Fp < 0 || c.Fpa < 0) return bad("flat observation too long");
    }
    {
        auto magic = [](int n) { return n > 1 ? (uint32_t)((1ull << 32) / (uint64_t)n) + 1u : 0u; };
        c.HW_magic = magic(c.HW); c.ww_magic = magic(c.win * c.win);
        c.Fa_magic = magic(c.Fa); c.Fpa_magic = magic(c.Fpa); c.Na_magic = magic(c.Na);
        c.win_magic = magic(c.win); c.win_dr32 = 32 / c.win; c.win_dc32 = 32 - c.win_dr32 * c.win;
    }
    c.tab_p = c.Fa; c.tab_pa = c.tab_p + c.Fp; c.tab_m = c.tab_pa + c.Fpa;
    c.tab_hoff = c.tab_m + c.Na;
    c.tab_seg = c.tab_hoff + 4 * c.P;
    memcpy(tb.w, prog_a, 2 * c.Fa); memcpy(tb.w + c.tab_p, prog_p, 2 * c.Fp);
    memcpy(tb.w + c.tab_pa, prog_pa, 2 * c.Fpa); memcpy(tb.w + c.tab_m, mask_prog, 2 * c.Na);
    {
        // mask segments (random policy): runs of consecutive mask entries of one slot with idx 0 .. count-1
        int n_seg = 0, si = 0;
        c.seg_lo[0] = 0;
        for (int j = 0; j < c.Na;) {
            const int slot = mask_prog[j] >> 8;
            int cnt = 0;
            while (j + cnt < c.Na && (mask_prog[j + cnt] >> 8) == slot && (mask_prog[j + cnt] & 255) == cnt) cnt++;
            // a multi-action subspace starts with its own NO-OP entry (slot MS_ONE): close the previous subspace there
            if (c.multi_action && slot == MS_ONE && n_seg > 0) c.seg_lo[++si] = n_seg;
            if (n_seg >= 64) return bad("too many action mask segments");
            tb.w[c.tab_seg + n_seg++] = (uint16_t)((cnt << 8) | slot);
            j += cnt;
        }
        c.seg_lo[++si] = n_seg;
        if (si != c.n_act_a) return bad("internal: mask segments do not match the action subspaces");
        c.tab_lut = (c.tab_seg + n_seg + 7) & ~7;   // 16-byte aligned (u16 words)
        float *lut = (float *)(tb.w + c.tab_lut);   // nibble -> four floats (bit k of the nibble -> element k)
        for (int k = 0; k < 16; k++) for (int j = 0; j < 4; j++) lut[4 * k + j] = (float)((k >> j) & 1);
        if (c.obs_bf16) {   // nibble -> four bfloat16 (8 bytes), in the same slot
            uint16_t *lut16 = tb.w + c.tab_lut;
            for (int k = 0; k < 16; k++) for (int j = 0; j < 4; j++) lut16[4 * k + j] = (uint16_t)(((k >> j) & 1) ? 0x3F80u : 0u);
        }
        c.tab_n = c.tab_lut + 128;
        // compacted transfer: every entry of the agents' flat program gets its index inside its class
        c.tab_cslot = c.tab_n;
        c.cf_n_sh = c.cf_n_ag = c.cf_n_cnt = 0;
        for (int j = 0; j < c.Fa; j++) {
            const int kind = AIE_FLAT_KIND(prog_a[j]);
            int &n = kind == FK_SHARED ? c.cf_n_sh : (kind == FK_AGENT ? c.cf_n_ag : c.cf_n_cnt);
            tb.w[c.tab_cslot + j] = (uint16_t)n++;
        }
        if (c.tab_cslot + c.Fa > TAB_WORDS) return bad("internal: table overflow");
    }
    // record layout
    {
        const int A = c.A, P = c.P;
        c.st_trade = ST_BUILDS + A;
        c.st_tax = c.has[COMP_TAX] ? c.st_trade + 8 * A : -1;
        c.n_stats = c.has[COMP_TAX] ? c.st_tax + ST_TAX_AGENT + 2 * A : c.st_trade + 8 * A;
        // Large envs (split) keep the rarely touched episode statistics with the other big sections in global memory.
        auto layout = [&](bool stats_last) {
            int off = HDR_WORDS * 4;
            auto take = [&](int bytes) { int o = off; off = align16(off + bytes); return o; };
            c.off_coin = take(8 * A); c.off_esc_coin = take(8 * A); c.off_labor = take(8 * A);
            c.off_bpay = take(8 * A); c.off_bskill = take(8 * A); c.off_bonus = take(8 * A);
            c.off_last_coin = take(8 * A); c.off_last_income = take(8 * A); c.off_last_marg = take(8 * A);
            c.off_util_prev = take(8 * (A + 1));
            c.off_inv = take(4 * 2 * A); c.off_esc = take(4 * 2 * A);
            c.off_loc = take(2 * 2 * A);
            c.off_n_orders = take(2 * A); c.off_bid_hist = take(2 * A * P); c.off_ask_hist = take(2 * A * P);
            c.off_rate_idx = take(16);
            c.off_cell = take(c.HW); c.off_owner = take(c.HW);
            c.obs_prefix_bytes = off;                  // [0, here): what the observation pass reads besides price_hist
            if (!stats_last) c.off_stats = take(8 * c.n_stats);
            c.off_mt = take(4 * 624);
            // Saez model: current bracket rates [16], their running average [16] and the rates the observations show
            // [16] (float64), kept across resets
            c.off_saez = (c.has[COMP_TAX] && c.tax_model == AIE_TAX_SAEZ) ? take(8 * 48) : 0;
            c.off_gauss = (c.reset_mode == 1 && (c.build_skill_dist == 2 || c.gather_skill_dist == 2 || c.dyn_layout)) ? take(16) : 0;
            c.off_split_skill = c.split_layout ? take(8 * A) : 0;
            c.keep_bytes = off - c.off_mt;
            c.off_price_hist = take(8 * 2 * A * P);
            c.off_orders = take(4 * 2 * A * c.K);
            if (stats_last) c.off_stats = take(8 * c.n_stats);
            c.rec_bytes = off;
        };
        layout(false);
        // Large records (deep order books, many agents): one CTA of four warps per env (mw = 4), the whole record resident in
        // shared memory.  Records too large even for that keep the two big, sparsely touched sections in HBM/L2 (split).
        c.mw = (c.rec_bytes > 24 * 1024) ? 4 : 1;
        c.split = (c.rec_bytes > 100 * 1024) ? 1 : 0;
        if (const char *v = getenv("AIE_MW")) { const int k = atoi(v); if (k == 1 || k == 4) c.mw = k; }          // tuning aids
        if (const char *v = getenv("AIE_SPLIT")) { const int k = atoi(v); if (k == 0 || k == 1) c.split = k; }
        if (c.split) layout(true);
        c.resident_bytes = c.split ? c.off_price_hist : c.rec_bytes;
        c.step_scratch_bytes = align16(8 * (2 * A + 4) + 16 * A + 7 * A + 16);
        {   // histogram offsets of the FK_MY / FK_AVAIL entries: i = (side * 2 + commodity) * P + level -> byte offset from
            // bid_hist of agent 0's counter (agent a adds a * P)
            for (int i = 0; i < 4 * P; i++) {
                const int side = i / (2 * P), r = i - side * 2 * P, cc = r / P, pl = r - cc * P;
                tb.w[c.tab_hoff + i] = (uint16_t)(side * (c.off_ask_hist - c.off_bid_hist) + cc * A * P + pl);
            }
        }
        // ---- observation staging (aie_obs.cuh: ObsScratch) ----
        const int ww = c.win * c.win, HW4 = (c.HW + 3) & ~3;
        const int units = (ww + 7) >> 3;
        c.wcu_magic = units > 1 ? (uint32_t)((1ull << 32) / (uint64_t)units) + 1u : 0u;
        c.pl_stride_a = 4 * ((ww + 31) / 32);
        c.pl_stride_p = 4 * ((c.HW + 31) / 32);
        int need[OB_COUNT];
        need[OB_NET_HIST] = align16(8 * (2 * P + 2));
        need[OB_SHF] = align16(4 * c.sh_count);
        need[OB_SC_A] = align16(4 * A * AS_COUNT);
        need[OB_LIM] = align16(A * MS_COUNT);
        need[OB_PSH] = 16;
        need[OB_LOCMAP] = align16(HW4 + 8);
        const bool whole_map = c.planner_spatial || c.full_obs;
        auto chunk_needs = [&](int ac) {
            need[OB_WI] = align16(std::max(ac * 2 * ww, c.full_obs ? 2 * HW4 : 0) + 16);
            need[OB_PL] = align16(std::max(ac * (c.M + 1) * c.pl_stride_a, whole_map ? c.M * c.pl_stride_p : 0) + 16);
            need[OB_BITS] = align16(4 * ((std::max(ac * (c.M + 1) * ww, whole_map ? c.M * c.HW : 0) + 31) / 32) + 16);
        };
        const int early_ids[] = {OB_NET_HIST, OB_SHF, OB_SC_A, OB_LIM, OB_PSH, OB_LOCMAP};
        const int late_ids[] = {OB_WI, OB_PL, OB_BITS};
        // Device placement.  One region of the env's shared memory becomes free during the pass: [off_mt, resident + step
        // scratch).  Its first part, the MT19937 key image, is free from the start (the key goes out as its own bulk group);
        // the rest - the other kept state, price history, order slots, step scratch - once the scalars are staged and the
        // record's write-back has been read (DevExec::record_stored).  Early buffers (used before that point) therefore sit in
        // the key image, or in extra memory when they do not fit; the late buffers follow them and run on into extra memory
        // behind the region as far as needed.
        const int mt_lo = c.off_mt, mt_hi = c.off_mt + 4 * 624;
        const int scr_lo = c.resident_bytes, scr_hi = c.resident_bytes + c.step_scratch_bytes;
        auto place = [&](int ac, bool commit) {
            chunk_needs(ac);
            int off[OB_COUNT];
            // early buffers: first fit, largest first, into the key image and then into the step scratch (dead as soon as the
            // dynamics are done and never part of the write-back); if one does not fit, all of them go to extra memory
            int order[6] = {OB_NET_HIST, OB_SHF, OB_SC_A, OB_LIM, OB_PSH, OB_LOCMAP};
            std::sort(order, order + 6, [&](int a, int b) { return need[a] > need[b]; });
            int cur_mt = mt_lo, cur_scr = scr_lo;
            bool early_fits = true;
            for (int id : order) {
                if (need[id] <= mt_hi - cur_mt) { off[id] = cur_mt; cur_mt += need[id]; }
                else if (need[id] <= scr_hi - cur_scr) { off[id] = cur_scr; cur_scr += need[id]; }
                else { early_fits = false; break; }
            }
            if (!early_fits) { cur_mt = mt_lo; cur_scr = scr_lo; }
            // late buffers: from the end of the early ones in the key image on, through the rest of the dead region (they
            // stop short of early buffers parked in the scratch) and on into extra memory behind it
            const int late_lo = cur_mt;
            const int late_hi = (early_fits && cur_scr > scr_lo) ? scr_lo : scr_hi;
            int cur = late_lo;
            for (int id : late_ids) { off[id] = cur; cur += need[id]; }
            int end = cur;
            int extra = 0;
            if (end > late_hi) {   // the overflow continues behind the whole region: shift what lies beyond late_hi
                const int shift = scr_hi - late_hi;   // 0, or the scratch bytes the early buffers occupy
                if (shift) {
                    // simplest correct placement: when the late block does not fit in front of the parked early buffers, put
                    // the whole late block behind the region
                    int c2 = scr_hi;
                    for (int id : late_ids) { off[id] = c2; c2 += need[id]; }
                    end = c2;
                }
                extra = end - scr_hi;
            }
            if (!early_fits) { int c2 = std::max(end, scr_hi); for (int id : early_ids) { off[id] = c2; c2 += need[id]; } extra = c2 - scr_hi; }
            if (commit) {
                for (int i = 0; i < OB_COUNT; i++) c.ob[i] = off[i];
                c.obs_extra_bytes = align16(extra);
                c.obs_alias_mt = early_fits ? 1 : 0;
            }
            return extra;
        };
        {
            // agents per window chunk: the largest count (<= 16) whose staging needs no more shared memory than one agent's
            const int base_extra = place(1, false);
            int best = 0;
            for (int ac = std::min(A, 16); ac >= 1; ac--)
                if (place(ac, false) <= base_extra) { best = ac; break; }
            c.ob_chunk = best ? best : std::min(A, 4);
            place(c.ob_chunk, true);
        }
        {   // staging apart from the record (ob_emu): everything in one separate allocation, nothing aliases
            chunk_needs(c.ob_chunk);
            int off = 0;
            for (int i = 0; i < OB_COUNT; i++) { c.ob_emu[i] = off; off += need[i]; }
            c.obs_scratch_bytes = off;
        }
    }
    return AIE_OK;
}

// The columns of the episode-metrics table: the keys of the reference's env.metrics for this config in the dict's
// insertion order (foundation/metrics.py builds the same dict), each with the MT_* op the metrics kernel evaluates there.
// Scenario keys first, then every component's in component order; keys a config does not have are left out.
inline void build_metric_layout(const DevCfg &c, std::vector<aie_metric_key> &keys, std::vector<uint32_t> &prog) {
    keys.clear(); prog.clear();
    auto add = [&](const std::string &k, int op, int arg, int is_int) {
        aie_metric_key m;
        memset(&m, 0, sizeof(m));
        snprintf(m.key, sizeof(m.key), "%s", k.c_str());
        m.is_int = is_int;
        keys.push_back(m);
        prog.push_back((uint32_t)op << 24 | (uint32_t)arg);
    };
    const int A = c.A;
    auto num =[](int i) { return std::to_string(i); };
    add("social/productivity", MT_PRODUCTIVITY, 0, 0);
    add("social/equality", MT_EQUALITY, 0, 0);
    add("social_welfare/coin_eq_times_productivity", MT_COIN_EQ_PROD, 0, 0);
    if (c.one_step) {   // one_step_economy.py:210-262
        add("social_welfare/inv_income_weighted_utility", MT_INV_W_UTIL, 0, 0);
        add("endow/avg_agent/Coin", MT_MEAN_COIN, 0, 0);
        add("endogenous/avg_agent/Labor", MT_MEAN_LABOR, 0, 0);
        add("util/avg_agent", MT_MEAN_UTIL, 0, 0);
        add("endow/p/Coin", MT_ZERO, 0, 1);
        add("util/p", MT_UTIL, A, 0);
    } else {            // layout_from_file.py:595-650
        add("social_welfare/inv_income_weighted_coin_endow", MT_INV_W_COIN, 0, 0);
        add("social_welfare/inv_income_weighted_utility", MT_INV_W_UTIL, 0, 0);
        for (int a = 0; a < A; a++) {
            add("endow/" + num(a) + "/Coin", MT_COIN, a, 0);
            add("endow/" + num(a) + "/Stone", MT_INV, 2 * a, 0);
            add("endow/" + num(a) + "/Wood", MT_INV, 2 * a + 1, 0);
            add("endogenous/" + num(a) + "/Labor", MT_LABOR, a, 0);
            add("util/" + num(a), MT_UTIL, a, 0);
        }
        for (const char *r : {"Coin", "Stone", "Wood"}) add(std::string("endow/p/") + r, MT_ZERO, 0, 0);
        add("util/p", MT_UTIL, A, 0);
        add("labor/weighted_cost", MT_WEIGHTED_COST, 0, 0);
        add("labor/warmup_integrator", MT_WARMUP_INT, 0, 1);
    }
    static const char *CN[2] = {"Stone", "Wood"}, *SIDE[2] = {"Sell", "Buy"};
    for (int i = 0; i < c.n_comp; i++) {
        if (c.comp[i] == COMP_BUILD) {   // build.py:198-222
            for (int a = 0; a < A; a++) add("Build/" + num(a) + "/n_builds", MT_N_BUILDS, a, 1);
            add("Build/total_builds", MT_TOTAL_BUILDS, 0, 1);
        } else if (c.comp[i] == COMP_CDA) {   // continuous_double_auction.py:585-641 (cost == income == price)
            for (int a = 0; a < A; a++)
                for (int cc = 0; cc < 2; cc++)
                    for (int side = 0; side < 2; side++) {
                        const std::string p = "Trade/" + num(a) + "/" + SIDE[side] + CN[cc] + "/";
                        const int idx = c.st_trade + ((a * 2 + cc) * 2 + side) * 2;
                        for (const char *k : {"price", "cost", "income"}) add(p + k, MT_TRADE_AVG, idx, 0);
                        add(p + "n_sales", MT_TRADE_N, idx, 1);
                    }
            add("Trade/n_trades", MT_N_TRADES, 0, 1);
        } else if (c.comp[i] == COMP_TAX) {   // redistribution.py:1141-1186
            // the reference keys its logs by "%03d" % int(cutoff): brackets that share a key are pooled, in first-seen order
            std::vector<std::pair<std::string, int>> groups;
            for (int b = 0; b < c.B; b++) {
                char k[32];
                snprintf(k, sizeof(k), "%03lld", (long long)c.cutoffs[b]);
                auto it = std::find_if(groups.begin(), groups.end(), [&](const std::pair<std::string, int> &g) { return g.first == k; });
                if (it == groups.end()) groups.push_back({k, 1 << b});
                else it->second |= 1 << b;
            }
            for (const auto &g : groups) {
                add("PeriodicTax/avg_bracket_rate/" + g.first, MT_BRACKET_RATE, g.second, 0);
                add("PeriodicTax/bracket_occupancy/" + g.first, MT_BRACKET_OCC, g.second, 0);
            }
            if (!c.disable_taxes) {
                add("PeriodicTax/avg_effective_tax_rate", MT_EFF_RATE, 0, 0);
                add("PeriodicTax/total_collected_taxes", MT_COLLECTED, 0, 0);
                add("PeriodicTax/avg_tax_rate/poorest", MT_TAX_POOREST, 0, 0);
                add("PeriodicTax/avg_tax_rate/richest", MT_TAX_RICHEST, 0, 0);
                // the running elasticity estimate lives in the host-side Saez estimator: the caller fills this column
                if (c.tax_model == AIE_TAX_SAEZ) add("PeriodicTax/saez/estimated_elasticity", MT_NAN, 0, 0);
            }
        }
    }
}

inline void fill_dims(const DevCfg &c, aie_dims &d) {
    memset(&d, 0, sizeof(d));
    d.n_envs = c.n_envs; d.n_agents = c.A; d.height = c.H; d.width = c.W;
    d.n_map_channels = c.M; d.window = c.win;
    d.flat_agent = c.Fa; d.flat_planner = c.Fp; d.flat_planner_agent = c.Fpa;
    d.mask_agent = c.Na; d.mask_planner = c.Np; d.n_act_agent = c.n_act_a; d.n_act_planner = c.n_act_p;
    d.state_bytes = c.rec_bytes;
    d.n_stats = c.n_stats; d.stats_trade = c.st_trade; d.stats_tax = c.st_tax;
    d.agent_map_elems = c.a_map_elems; d.agent_idx_elems = c.a_idx_elems;
    const int fb = c.obs_bf16 ? 2 : 4;   // bytes per element of the float tensors
    long long obs = (long long)c.A * (c.a_map_elems * fb + c.a_idx_elems * 2 + c.Fa * fb + c.Na * fb) + c.Fp * fb + c.A * c.Fpa * fb +
                    c.Np * fb + fb + (c.planner_spatial ? (c.M * c.HW * fb + 2 * c.HW * 2) : 0);
    long long io = 8 * (c.A + 1) + 4 + 4 * (c.A * c.n_act_a + c.n_act_p);
    d.algorithmic_bytes_per_env_step = (int32_t)(obs + io + 2LL * c.rec_bytes);
}

struct FieldDesc { const char *name; int off, eb, flt, sgn, nd, s0, s1, s2; };

inline int lookup_field(const DevCfg &c, const char *name, aie_field *f) {
    const int A = c.A, P = c.P;
    const FieldDesc tab[] = {
        {"t", HDR_T * 4, 4, 0, 1, 0, 0, 0, 0}, {"tax_pos", HDR_TAX_POS * 4, 4, 0, 1, 0, 0, 0, 0},
        {"completions", HDR_COMPLETIONS * 4, 4, 0, 1, 0, 0, 0, 0}, {"auto_warmup", HDR_AUTO_WARMUP * 4, 4, 0, 1, 0, 0, 0, 0},
        {"mt_pos", HDR_MT_POS * 4, 4, 0, 1, 0, 0, 0, 0}, {"episodes", HDR_EPISODES * 4, 4, 0, 1, 0, 0, 0, 0},
        {"stats", c.off_stats, 8, 1, 1, 1, c.n_stats, 0, 0}, {"saez_n", HDR_SAEZ_N * 4, 4, 0, 1, 0, 0, 0, 0},
        {"saez_rates", c.off_saez, 8, 1, 1, 1, 16, 0, 0}, {"saez_avg_rates", c.off_saez + 128, 8, 1, 1, 1, 16, 0, 0},
        {"saez_obs_rates", c.off_saez + 256, 8, 1, 1, 1, 16, 0, 0}, {"util_prev", c.off_util_prev, 8, 1, 1, 1, A + 1, 0, 0},
        {"gauss_state", c.off_gauss, 8, 1, 1, 1, 2, 0, 0},
        {"coin", c.off_coin, 8, 1, 1, 1, A, 0, 0}, {"esc_coin", c.off_esc_coin, 8, 1, 1, 1, A, 0, 0},
        {"labor", c.off_labor, 8, 1, 1, 1, A, 0, 0}, {"build_payment", c.off_bpay, 8, 1, 1, 1, A, 0, 0},
        {"build_skill", c.off_bskill, 8, 1, 1, 1, A, 0, 0}, {"bonus_gather_prob", c.off_bonus, 8, 1, 1, 1, A, 0, 0},
        {"last_coin", c.off_last_coin, 8, 1, 1, 1, A, 0, 0}, {"last_income", c.off_last_income, 8, 1, 1, 1, A, 0, 0},
        {"last_marg", c.off_last_marg, 8, 1, 1, 1, A, 0, 0}, {"util_prev", c.off_util_prev, 8, 1, 1, 1, A + 1, 0, 0},
        {"price_hist", c.off_price_hist, 8, 1, 1, 3, 2, A, P}, {"inv", c.off_inv, 4, 0, 1, 2, A, 2, 0},
        {"esc", c.off_esc, 4, 0, 1, 2, A, 2, 0}, {"loc", c.off_loc, 2, 0, 1, 2, A, 2, 0},
        {"n_orders", c.off_n_orders, 1, 0, 0, 2, 2, A, 0}, {"bid_hist", c.off_bid_hist, 1, 0, 0, 3, 2, A, P},
        {"ask_hist", c.off_ask_hist, 1, 0, 0, 3, 2, A, P}, {"rate_idx", c.off_rate_idx, 1, 0, 0, 1, 16, 0, 0},
        {"cell", c.off_cell, 1, 0, 0, 2, c.H, c.W, 0}, {"owner", c.off_owner, 1, 0, 1, 2, c.H, c.W, 0},
        {"orders", c.off_orders, 4, 0, 0, 3, 2, A, c.K}, {"mt_key", c.off_mt, 4, 0, 0, 1, 624, 0, 0},
    };
    for (const FieldDesc &t : tab)
        if (!strcmp(t.name, name)) {
            if (!strncmp(name, "saez_", 5) && name[5] != 'n' && !c.off_saez) return AIE_EINVAL;  // no Saez section in this config
            if (!strcmp(name, "gauss_state") && !c.off_gauss) return AIE_EINVAL;
            f->offset = t.off; f->elem_bytes = t.eb; f->is_float = t.flt; f->is_signed = t.sgn; f->ndim = t.nd;
            f->shape[0] = t.s0; f->shape[1] = t.s1; f->shape[2] = t.s2; f->shape[3] = 0;
            return AIE_OK;
        }
    return AIE_EINVAL;
}

// Pack env i of a host reset snapshot into one record (books empty, escrow/labor zero; tax trackers and
// metric_0 are finished on the device by finish_reset_env).
inline int pack_record(const DevCfg &c, const aie_host_state &hs, int i, uint8_t *rec, std::string &err) {
    const int A = c.A, HW = c.HW;
    memset(rec, 0, c.rec_bytes);
    int32_t *hdr = (int32_t *)rec;
    hdr[HDR_T] = 0; hdr[HDR_TAX_POS] = 1;
    hdr[HDR_COMPLETIONS] = hs.completions ? hs.completions[i] : 0;
    hdr[HDR_MT_POS] = hs.mt_pos[i];
    if (hs.mt_pos[i] < 0 || hs.mt_pos[i] > 624) { err = "mt_pos out of range"; return AIE_EINVAL; }
    double *coin = (double *)(rec + c.off_coin), *bpay = (double *)(rec + c.off_bpay),
           *bskill = (double *)(rec + c.off_bskill), *bonus = (double *)(rec + c.off_bonus);
    int32_t *inv = (int32_t *)(rec + c.off_inv);
    int16_t *loc = (int16_t *)(rec + c.off_loc);
    uint8_t *cell = rec + c.off_cell;
    int8_t *owner = (int8_t *)(rec + c.off_owner);
    for (int k = 0; k < HW; k++) {
        size_t g = (size_t)i * HW + k;
        uint8_t b = 0;
        if (hs.stone[g]) b |= CELL_STONE;
        if (hs.wood[g]) b |= CELL_WOOD;
        if (hs.stone_src[g]) b |= CELL_STONE_SRC;
        if (hs.wood_src[g]) b |= CELL_WOOD_SRC;
        if (hs.water && hs.water[g]) b |= CELL_WATER;
        cell[k] = b; owner[k] = -1;
    }
    for (int a = 0; a < A; a++) {
        size_t g = (size_t)i * A + a;
        int r = hs.loc[2 * g], cc = hs.loc[2 * g + 1];
        if (r < 0 || r >= c.H || cc < 0 || cc >= c.W) { err = "agent location outside the world"; return AIE_EINVAL; }
        loc[2 * a] = (int16_t)r; loc[2 * a + 1] = (int16_t)cc;
        coin[a] = hs.coin[g];
        if (!(hs.coin[g] >= 0.0)) { err = "negative starting coin"; return AIE_EINVAL; }
        inv[2 * a] = hs.inv_stone ? hs.inv_stone[g] : 0;
        inv[2 * a + 1] = hs.inv_wood ? hs.inv_wood[g] : 0;
        bpay[a] = hs.build_payment[g]; bskill[a] = hs.build_skill[g]; bonus[a] = hs.bonus_gather_prob[g];
    }
    uint32_t *orders = (uint32_t *)(rec + c.off_orders);
    for (int k = 0; k < 2 * A * c.K; k++) orders[k] = ORDER_EMPTY;
    memcpy(rec + c.off_mt, hs.mt_key + (size_t)i * 624, 624 * 4);
    if (c.off_split_skill) {
        if (!hs.split_skill) { err = "split_layout device reset needs aie_host_state.split_skill"; return AIE_EINVAL; }
        memcpy(rec + c.off_split_skill, hs.split_skill + (size_t)i * c.A, 8 * (size_t)c.A);
    }
    if (c.off_gauss) {
        double *g = (double *)(rec + c.off_gauss);
        g[0] = hs.gauss_val ? hs.gauss_val[i] : 0.0;
        g[1] = (hs.gauss_has && hs.gauss_has[i]) ? 1.0 : 0.0;
    }
    return AIE_OK;
}

// Unpack a record for tests (aie_read_state).
inline void unpack_record(const DevCfg &c, const uint8_t *rec, const aie_state_dump &d) {
    const int A = c.A, P = c.P, HW = c.HW, K = c.K;
    const int32_t *hdr = (const int32_t *)rec;
    const int t = hdr[HDR_T];
    if (d.cell) memcpy(d.cell, rec + c.off_cell, HW);
    if (d.owner) memcpy(d.owner, rec + c.off_owner, HW);
    if (d.loc) memcpy(d.loc, rec + c.off_loc, 4 * A);
    if (d.coin) memcpy(d.coin, rec + c.off_coin, 8 * A);
    if (d.esc_coin) memcpy(d.esc_coin, rec + c.off_esc_coin, 8 * A);
    if (d.labor) memcpy(d.labor, rec + c.off_labor, 8 * A);
    if (d.inv) memcpy(d.inv, rec + c.off_inv, 8 * A);
    if (d.esc) memcpy(d.esc, rec + c.off_esc, 8 * A);
    if (d.last_coin) memcpy(d.last_coin, rec + c.off_last_coin, 8 * A);
    if (d.last_income) memcpy(d.last_income, rec + c.off_last_income, 8 * A);
    if (d.last_marg) memcpy(d.last_marg, rec + c.off_last_marg, 8 * A);
    if (d.price_hist) memcpy(d.price_hist, rec + c.off_price_hist, 8 * 2 * A * P);
    for (int i = 0; i < 2 * A; i++) if (d.n_orders) d.n_orders[i] = rec[c.off_n_orders + i];
    for (int i = 0; i < 2 * A * P; i++) {
        if (d.bid_hist) d.bid_hist[i] = rec[c.off_bid_hist + i];
        if (d.ask_hist) d.ask_hist[i] = rec[c.off_ask_hist + i];
    }
    if (d.tax_pos) *d.tax_pos = hdr[HDR_TAX_POS];
    if (d.rate_idx) for (int b = 0; b < c.B; b++) d.rate_idx[b] = rec[c.off_rate_idx + b];
    if (d.mt_key) memcpy(d.mt_key, rec + c.off_mt, 624 * 4);
    if (d.mt_pos) *d.mt_pos = hdr[HDR_MT_POS];
    if (d.t) *d.t = t;
    if (d.completions) *d.completions = hdr[HDR_COMPLETIONS];
    if (d.stats) memcpy(d.stats, rec + c.off_stats, 8 * c.n_stats);
    if (d.util_prev) memcpy(d.util_prev, rec + c.off_util_prev, 8 * (A + 1));
    if (d.auto_warmup) *d.auto_warmup = hdr[HDR_AUTO_WARMUP];
    if (d.book_rows && d.book_count) {
        const uint32_t *orders = (const uint32_t *)(rec + c.off_orders);
        struct Row { int agent, price, life; };
        for (int cc = 0; cc < 2; cc++)
            for (int side = 0; side < 2; side++) {
                std::vector<Row> rows;
                for (int a = 0; a < A; a++)
                    for (int k = 0; k < K; k++) {
                        uint32_t o = orders[(cc * A + a) * K + k];
                        if (o == ORDER_EMPTY || (int)(o & 1u) != side) continue;
                        // the reference increments lifetimes at the end of the step (remove_expired_orders)
                        rows.push_back(Row{a, (int)((o >> 1) & 127u), t - (int)(o >> 8) + 1});
                    }
                std::stable_sort(rows.begin(), rows.end(), [side](const Row &x, const Row &y) {
                    if (x.price != y.price) return side == 0 ? x.price > y.price : x.price < y.price;
                    if (x.life != y.life) return x.life > y.life;
                    return x.agent < y.agent;
                });
                int n = (int)rows.size();
                d.book_count[cc * 2 + side] = n;
                int32_t *out = d.book_rows + (size_t)(cc * 2 + side) * d.book_cap * 3;
                for (int i = 0; i < n && i < d.book_cap; i++) { out[3 * i] = rows[i].agent; out[3 * i + 1] = rows[i].price; out[3 * i + 2] = rows[i].life; }
            }
    }
}

}  // namespace aie
