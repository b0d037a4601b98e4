"""`foundation` — same entry points as ai_economist.foundation (foundation/__init__.py:7-18):
six registries and make_env_instance(scenario_name, **kwargs)."""
from . import agents as _agents_mod
from . import components as _components_mod
from . import entities as _entities_mod
from . import scenarios as _scenarios_mod
from .batched_env import BatchedFoundationEnv
from . import covid19 as _covid_mod  # noqa: F401  (registers the COVID-19 scenario and its components)

agents = _agents_mod.agent_registry
components = _components_mod.component_registry
endogenous = _entities_mod.endogenous_registry
landmarks = _entities_mod.landmark_registry
resources = _entities_mod.resource_registry
scenarios = _scenarios_mod.scenario_registry


def make_env_instance(scenario_name, **kwargs):
    """Same call as the reference; extra kwargs: n_envs (default 1), device ("cuda:0"), seeds, auto_reset, obs_dtype,
    final_obs, and
    reference_api (or AIE_REFERENCE_API=1 in the environment): wrap replica 0 in adapters.ReferenceApiEnv, whose
    reset()/step() take and return the reference's nested numpy dictionaries, so tutorial code runs unchanged."""
    import os
    ref_api = kwargs.pop("reference_api", None)
    if ref_api is None:
        ref_api = os.environ.get("AIE_REFERENCE_API", "0") not in ("", "0")
    if ref_api:
        from ..adapters import ReferenceApiEnv
        if getattr(scenarios.get(scenario_name), "env_class", None) is not None:
            raise NotImplementedError("reference_api covers the gather-trade-build scenarios; the COVID-19 env already "
                                      "returns the reference's collated layout (with a leading env axis)")
        kwargs.setdefault("auto_reset", False)   # the caller resets explicitly, like the reference's loops do
        return ReferenceApiEnv(make_env_instance(scenario_name, reference_api=False, **kwargs))
    scenario_cls = scenarios.get(scenario_name)
    env_class = getattr(scenario_cls, "env_class", None)
    if env_class is not None:  # scenarios with their own device path (COVID-19)
        return env_class(**kwargs)
    return BatchedFoundationEnv(scenario_cls, **kwargs)
