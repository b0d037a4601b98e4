"""Plumbing shared by the batched envs' `state_dict()` / `load_state_dict()`: the configuration a checkpoint was taken
from, and copies of device buffers in and out (torch tensors on the CUDA backend, numpy arrays on numpy backends)."""
import copy

import numpy as np

FORMAT_VERSION = 1   # of the dict state_dict() returns; load_state_dict() refuses any other


def plain(v):
    """v with numpy scalars / arrays and tuples turned into Python values and lists (for comparing configurations)."""
    if isinstance(v, dict):
        return {str(k): plain(x) for k, x in v.items()}
    if isinstance(v, (list, tuple, np.ndarray)):
        return [plain(x) for x in (v.tolist() if isinstance(v, np.ndarray) else v)]
    if isinstance(v, np.generic):
        return v.item()
    return v


def check_config(sd, config):
    """ValueError naming the first field of `config` in which the checkpoint `sd` differs."""
    if not isinstance(sd, dict) or "format_version" not in sd:
        raise ValueError("load_state_dict: not an env state dict (no format_version)")
    if sd["format_version"] != FORMAT_VERSION:
        raise ValueError("load_state_dict: format_version %r, this library reads %d" % (sd["format_version"],
                                                                                         FORMAT_VERSION))
    theirs = sd.get("config", {})
    for k, v in config.items():   # in order: the numeric spec comes last, so a named option is reported by its name
        a, b = plain(theirs.get(k)), plain(v)
        if a == b:
            continue
        if isinstance(a, dict) and isinstance(b, dict):
            sub = next(s for s in list(b) + list(a) if a.get(s) != b.get(s))
            k, a, b = "%s[%r]" % (k, sub), a.get(sub), b.get(sub)
        raise ValueError("load_state_dict: the checkpoint was taken from a different configuration: %s differs "
                         "(checkpoint %s, this env %s)" % (k, _short(a), _short(b)))


def _short(v):
    s = repr(plain(v))
    return s if len(s) <= 200 else s[:200] + "..."


def refuse_mid_rollout(env, fn):
    if env._rollout is not None and env._stepper.rollout_slot != 0:
        raise ValueError("%s: a bound rollout is checkpointed only at slot 0 (before its first step or right after "
                         "restart_rollout()); its slots are the trainer's data, not env state" % fn)


def snapshot(buf):
    """A copy of a buffer on its own backend."""
    return buf.copy() if isinstance(buf, np.ndarray) else buf.detach().clone()


def copy_into(dst, src, name):
    """dst[...] = src, same shape and element type required (ValueError naming the buffer otherwise)."""
    if isinstance(dst, np.ndarray):
        s = src if isinstance(src, np.ndarray) else src.detach().cpu().numpy()
        if s.dtype != dst.dtype or s.shape != dst.shape:
            raise ValueError("load_state_dict: buffer %s is %s %s, this env's is %s %s"
                             % (name, s.dtype, s.shape, dst.dtype, dst.shape))
        dst[...] = s
        return
    import torch
    s = torch.as_tensor(src) if isinstance(src, np.ndarray) else src
    if s.dtype != dst.dtype or tuple(s.shape) != tuple(dst.shape):
        raise ValueError("load_state_dict: buffer %s is %s %s, this env's is %s %s"
                         % (name, s.dtype, tuple(s.shape), dst.dtype, tuple(dst.shape)))
    dst.copy_(s)


def host_copy(v):
    """A deep copy of host-side Python state (lists, dicts, numpy arrays)."""
    return copy.deepcopy(v)
