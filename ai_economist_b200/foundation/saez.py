"""Host half of the Saez tax model (PeriodicBracketTax(tax_model="saez"), components/redistribution.py:437-823).

Device/host hybrid (SURVEY 8f row 3): the step kernel enacts taxes with whatever bracket rates sit in the "saez_rates"
field of an env's record, counts the (income, marginal rate) samples it has produced ("saez_n") and, while fewer than
500 exist, draws the reference's uniform random warm-up rates from the env's own numpy stream.  Once per tax period -
after the step that closed a period, i.e. right before the step whose tax_cycle_pos is 1 - this module appends the
period's samples to the replica's buffer and, when the buffer is full, evaluates the Saez formula (elasticity
regression, binned welfare weights / Pareto parameters, bracketisation) in float64 numpy exactly in the order the
reference does, then writes the new rates and their running average back into the record.

`SaezEstimator` restates the reference's estimator for ONE env, numpy call by numpy call; `SaezBatch` is the same
arithmetic over a leading replica axis and is what `SaezHost` runs (tests/test_saez_batch.py pins it to the per-replica
version at 1e-10; the per-replica version is pinned on a 790-step reference trace).
"""
import numpy as np

BUFFER_SIZE = 500      # redistribution.py:276
N_BINS = 100           # :284


class SaezEstimator:
    def __init__(self, cutoffs, rate_min, rate_max, pareto_weight_type="inverse_income", fixed_elas=None):
        self.cutoffs = np.asarray(cutoffs, np.float64)
        self.B = len(self.cutoffs)
        self.bracket_sizes = np.concatenate([self.cutoffs, [np.inf]])[1:] - self.cutoffs   # :216-219
        self.rate_min, self.rate_max = float(rate_min), float(rate_max)
        assert pareto_weight_type in ("inverse_income", "uniform")
        self.pareto_weight_type = pareto_weight_type
        self.fixed_elas = None if fixed_elas is None else float(fixed_elas)
        self.edges = np.linspace(0, self.cutoffs[-1], N_BINS + 1)                          # :286-288
        self.bin_sizes = np.concatenate([self.edges[1:] - self.edges[:-1], [np.inf]])
        self.elas_tm1, self.elas_t, self.log_z0_tm1, self.log_z0_t = 0.5, 0.5, 0.0, 0.0    # :262-266
        self.running_avg = np.zeros(self.B)
        self.buffer = []                                                                    # [[income, marginal rate], ...]

    # -- the period's samples (:535-544) --------------------------------------------------------------
    def add_samples(self, incomes, marginal_rates):
        for z, tau in zip(incomes, marginal_rates):
            self.buffer.append([float(z), float(tau)])
        if len(self.buffer) > BUFFER_SIZE:
            del self.buffer[:len(self.buffer) - BUFFER_SIZE]

    @property
    def ready(self):
        return len(self.buffer) >= BUFFER_SIZE

    # -- elasticity (:549-599): OLS of log income on log(1 - rate), exponentially smoothed ------------------
    def _elasticity(self, data):
        keep = (data[:, 0] > 0) & (data[:, 1] < 1)
        zs, taus = data[keep, 0], data[keep, 1]
        if len(zs) < 10 or np.std(taus) < 1e-6:
            return float(self.elas_tm1), float(self.log_z0_tm1)
        x = np.log(np.maximum(1 - taus, 1e-9))
        X = np.stack([x, np.ones_like(x)]).T
        Y = np.log(np.maximum(zs, 1e-9))
        elas, log_z0 = np.linalg.inv(X.T.dot(X)).T.dot(X.T.dot(Y))
        return (1 - 0.98) * np.maximum(elas, 0.0) + 0.98 * self.elas_tm1, log_z0

    # -- binned welfare weights g(z) and Pareto parameters a(z) (:601-754) ---------------------------------
    def _pareto_weight(self, z):
        return np.ones_like(z) if self.pareto_weight_type == "uniform" else 1.0 / np.maximum(1, z)

    def _binned(self, incomes):
        counts, lefts = np.histogram(incomes, bins=self.edges)
        below, above = incomes[incomes < lefts[0]], incomes[incomes > lefts[-1]]
        n_total = np.sum(counts) + len(below) + len(above)
        pz = np.array([c / n_total for c in counts] + [len(above) / n_total])
        cum = [pz[0] + len(below) / n_total]
        for p in pz[1:]:
            cum.append(min(max(cum[-1] + p, 0), 1.0))
        cum = np.array(cum)
        # g(z): average normalised Pareto weight of everyone at or above z, bin-centred
        w_below = np.sum(self._pareto_weight(np.maximum(below, 0))) if len(below) else 0
        w_above = np.sum(self._pareto_weight(above)) if len(above) else 0
        w_bin = counts * self._pareto_weight(0.5 * (lefts[:-1] + lefts[1:]))
        norm = w_bin.sum() + w_below + w_above + 1e-9
        dens = np.concatenate([w_bin, [w_above]]) / norm
        g_geq = np.cumsum(dens[::-1])[::-1] / (np.cumsum(pz[::-1])[::-1] + 1e-9)
        gz = np.concatenate([0.5 * (g_geq[:-1] + g_geq[1:]), [g_geq[-1]]])
        # a(z) = z p(z) / P(Z >= z), per unit of bin width; the open top bin uses the mean income above the cutoff
        p_geq = 1 - cum + 0.5 * pz
        az = []
        for i in range(N_BINS):
            if pz[i] == 0:
                az.append(np.nan)
            else:
                z = 0.5 * (lefts[i] + lefts[i + 1])
                az.append(z * pz[i] / (min(max(p_geq[i], 0), 1) + 1e-9) / (lefts[i + 1] - lefts[i]))
        if len(above):
            m = np.mean(above)
            az.append(m / (m - lefts[-1] + 1e-9))
        else:
            az.append(0.0)
        return gz, np.array(az)

    # -- marginal rates per bin (:756-785), empty bins linearly interpolated ------------------------------
    @staticmethod
    def _bin_rates(gz, az, elas):
        taus = (1.0 - gz) / (1.0 - gz + az * elas + 1e-9)
        last_rate, last_i = 0.0, -1
        for i, tau in enumerate(taus):
            if np.isnan(tau):
                continue
            if i - last_i > 1:
                assert i != 0
                gap = list(range(last_i + 1, i))
                for k, r in zip(gap, np.linspace(last_rate, tau, len(gap) + 2)[1:-1]):
                    taus[k] = r
            last_rate, last_i = float(tau), i
        return taus

    # -- average marginal rate inside each tax bracket (:787-823) ------------------------------------------
    def _bracketize(self, bin_rates):
        out, last_total = [], 0
        for b, income in enumerate(self.cutoffs[1:]):
            due = np.maximum(0, np.sum(bin_rates * np.minimum(self.bin_sizes, np.maximum(0, income - self.edges))))
            out.append((due - last_total) / self.bracket_sizes[b])
            last_total = due
        out.append(bin_rates[-1])
        return np.array(out)

    def new_period_rates(self, rate_max=None):
        """compute_and_set_new_period_rates_from_saez_formula (:437-511) for a full buffer -> bracket rates [B].
        rate_max: curr_rate_max (:390-394) - the annealed maximum of the running episode under a tax_annealing_schedule."""
        data = np.array(self.buffer)
        self.elas_tm1, self.log_z0_tm1 = float(self.elas_t), float(self.log_z0_t)
        elas_t, log_z0_t = self._elasticity(data)
        self.elas_t, self.log_z0_t = float(elas_t), float(log_z0_t)
        if self.fixed_elas is not None:
            elas_t = self.fixed_elas
        gz, az = self._binned(data[:, 0])
        rates = np.clip(self._bracketize(self._bin_rates(gz, az, elas_t)), self.rate_min,
                        self.rate_max if rate_max is None else float(rate_max))
        self.running_avg = self.running_avg * 0.99 + rates * 0.01
        return rates


class SaezBatch:
    """The same estimator for E replicas at once: every numpy call of SaezEstimator becomes one call over a leading
    replica axis (sample buffers [E, 500, 2] kept in arrival order, masked sums for the regression, one bincount for the
    histograms, the cumulative / interpolation recurrences run over the 101 bins with vector state).  Agrees with the
    per-replica estimator to float64 rounding of the reordered sums (tests/test_saez_batch.py: <= 1e-10 relative); at
    8 192 replicas a tax period costs 0.55 s instead of 4.8 s in the build container."""

    def __init__(self, n, cutoffs, rate_min, rate_max, pareto_weight_type="inverse_income", fixed_elas=None):
        one = SaezEstimator(cutoffs, rate_min, rate_max, pareto_weight_type, fixed_elas)
        self.n, self.B = int(n), one.B
        self.cutoffs, self.bracket_sizes, self.edges, self.bin_sizes = one.cutoffs, one.bracket_sizes, one.edges, one.bin_sizes
        self.rate_min, self.rate_max = one.rate_min, one.rate_max
        self.pareto_weight_type, self.fixed_elas = one.pareto_weight_type, one.fixed_elas
        self.elas_tm1, self.elas_t = np.full(n, 0.5), np.full(n, 0.5)
        self.log_z0_tm1, self.log_z0_t = np.zeros(n), np.zeros(n)
        self.running_avg = np.zeros((n, self.B))
        self.buf = np.zeros((n, BUFFER_SIZE, 2))
        self.count = np.zeros(n, np.int64)     # samples held (<= BUFFER_SIZE)
        self.start = np.zeros(n, np.int64)     # ring position of the oldest sample

    # -- samples ------------------------------------------------------------------------------------------
    def add_samples(self, rows, incomes, marginal_rates):
        """rows: replica indices [R]; incomes / marginal_rates: [R, A] (one tax day)."""
        rows = np.asarray(rows, np.int64)
        A = incomes.shape[1]
        for j in range(A):   # A is small; each pass appends one sample per replica
            full = self.count[rows] >= BUFFER_SIZE
            pos = np.where(full, self.start[rows], (self.start[rows] + self.count[rows]) % BUFFER_SIZE)
            self.buf[rows, pos, 0] = incomes[:, j]
            self.buf[rows, pos, 1] = marginal_rates[:, j]
            self.start[rows] = np.where(full, (self.start[rows] + 1) % BUFFER_SIZE, self.start[rows])
            self.count[rows] = np.minimum(self.count[rows] + 1, BUFFER_SIZE)

    def ready(self, rows):
        return self.count[np.asarray(rows, np.int64)] >= BUFFER_SIZE

    def _data(self, rows):
        idx = (self.start[rows][:, None] + np.arange(BUFFER_SIZE)[None]) % BUFFER_SIZE     # arrival order
        return self.buf[rows[:, None], idx]

    # -- the formula, vectorised over the rows -----------------------------------------------------------------
    def _pareto_weight(self, z):
        return np.ones_like(z) if self.pareto_weight_type == "uniform" else 1.0 / np.maximum(1, z)

    def _elasticity(self, rows, data):
        keep = (data[:, :, 0] > 0) & (data[:, :, 1] < 1)
        n = keep.sum(axis=1)
        nn = np.maximum(n, 1)
        taus = np.where(keep, data[:, :, 1], 0.0)
        mean_tau = taus.sum(axis=1) / nn
        std_tau = np.sqrt(np.where(keep, (data[:, :, 1] - mean_tau[:, None]) ** 2, 0.0).sum(axis=1) / nn)
        x = np.where(keep, np.log(np.maximum(1 - np.where(keep, data[:, :, 1], 0.0), 1e-9)), 0.0)
        y = np.where(keep, np.log(np.maximum(np.where(keep, data[:, :, 0], 1.0), 1e-9)), 0.0)
        xtx = np.zeros((len(rows), 2, 2))
        xtx[:, 0, 0] = (x * x).sum(axis=1); xtx[:, 0, 1] = xtx[:, 1, 0] = x.sum(axis=1); xtx[:, 1, 1] = n
        xty = np.stack([(x * y).sum(axis=1), y.sum(axis=1)], axis=1)
        ok = (n >= 10) & (std_tau >= 1e-6)
        safe = np.where(ok[:, None, None], xtx, np.eye(2)[None])
        beta = np.einsum("eji,ej->ei", np.linalg.inv(safe), xty)          # inv(X'X).T @ (X'Y)
        elas = np.where(ok, (1 - 0.98) * np.maximum(beta[:, 0], 0.0) + 0.98 * self.elas_tm1[rows], self.elas_tm1[rows])
        log_z0 = np.where(ok, beta[:, 1], self.log_z0_tm1[rows])
        return elas, log_z0

    def _binned(self, incomes):
        R = incomes.shape[0]
        lefts = self.edges
        below, above = incomes < lefts[0], incomes > lefts[-1]
        inside = ~(below | above)
        idx = np.clip(np.searchsorted(lefts, incomes, side="right") - 1, 0, N_BINS - 1)    # np.histogram's binning
        flat = (np.arange(R)[:, None] * N_BINS + idx)[inside]
        counts = np.bincount(flat, minlength=R * N_BINS).reshape(R, N_BINS).astype(np.float64)
        n_below, n_above = below.sum(axis=1), above.sum(axis=1)
        n_total = counts.sum(axis=1) + n_below + n_above
        pz = np.concatenate([counts / n_total[:, None], (n_above / n_total)[:, None]], axis=1)      # [R, 101]
        cum = np.zeros_like(pz)
        cum[:, 0] = pz[:, 0] + n_below / n_total
        for i in range(1, N_BINS + 1):
            cum[:, i] = np.minimum(np.maximum(cum[:, i - 1] + pz[:, i], 0), 1.0)
        w_below = np.where(below, self._pareto_weight(np.maximum(np.where(below, incomes, 0.0), 0)), 0.0).sum(axis=1)
        w_above = np.where(above, self._pareto_weight(np.where(above, incomes, 1.0)), 0.0).sum(axis=1)
        w_bin = counts * self._pareto_weight(0.5 * (lefts[:-1] + lefts[1:]))[None]
        norm = w_bin.sum(axis=1) + w_below + w_above + 1e-9
        dens = np.concatenate([w_bin, w_above[:, None]], axis=1) / norm[:, None]
        g_geq = np.cumsum(dens[:, ::-1], axis=1)[:, ::-1] / (np.cumsum(pz[:, ::-1], axis=1)[:, ::-1] + 1e-9)
        gz = np.concatenate([0.5 * (g_geq[:, :-1] + g_geq[:, 1:]), g_geq[:, -1:]], axis=1)
        p_geq = 1 - cum + 0.5 * pz
        mid, width = 0.5 * (lefts[:-1] + lefts[1:]), lefts[1:] - lefts[:-1]
        with np.errstate(divide="ignore", invalid="ignore"):
            az_bins = mid[None] * pz[:, :N_BINS] / (np.minimum(np.maximum(p_geq[:, :N_BINS], 0), 1) + 1e-9) / width[None]
        az_bins = np.where(pz[:, :N_BINS] == 0, np.nan, az_bins)
        m = np.where(above, incomes, 0.0).sum(axis=1) / np.maximum(n_above, 1)
        az_top = np.where(n_above > 0, m / (m - lefts[-1] + 1e-9), 0.0)
        return gz, np.concatenate([az_bins, az_top[:, None]], axis=1)

    @staticmethod
    def _bin_rates(gz, az, elas):
        with np.errstate(invalid="ignore"):
            taus = (1.0 - gz) / (1.0 - gz + az * elas[:, None] + 1e-9)
        R, n = taus.shape
        valid = ~np.isnan(taus)
        pos = np.arange(n)[None]
        prev_i = np.maximum.accumulate(np.where(valid, pos, -1), axis=1)                     # last valid index <= k
        next_i = np.minimum.accumulate(np.where(valid, pos, n)[:, ::-1], axis=1)[:, ::-1]    # first valid index >= k
        rows = np.arange(R)[:, None]
        a = np.where(prev_i >= 0, taus[rows, np.maximum(prev_i, 0)], 0.0)                    # virtual (index -1, rate 0)
        b = taus[rows, np.minimum(next_i, n - 1)]
        step = (b - a) / np.maximum(next_i - prev_i, 1)                                      # np.linspace's step
        return np.where(valid, taus, (pos - prev_i) * step + a)

    def _bracketize(self, bin_rates):
        out = np.zeros((bin_rates.shape[0], self.B))
        last_total = np.zeros(bin_rates.shape[0])
        for b, income in enumerate(self.cutoffs[1:]):
            span = np.minimum(self.bin_sizes, np.maximum(0, income - self.edges))
            with np.errstate(invalid="ignore"):
                due = np.maximum(0, np.sum(bin_rates * span[None], axis=1))
            out[:, b] = (due - last_total) / self.bracket_sizes[b]
            last_total = due
        out[:, -1] = bin_rates[:, -1]
        return out

    CHUNK = 256   # replicas per pass: keeps the [chunk, 500] temporaries inside the CPU caches

    def new_period_rates(self, rows, rate_max=None):
        """Rates [R, B] of the replicas in `rows` (all with a full buffer); updates their smoothed state.  rate_max [R]:
        every replica's curr_rate_max (tax annealing), default the component's rate_max."""
        rows = np.asarray(rows, np.int64)
        cap = np.full(len(rows), self.rate_max) if rate_max is None else np.asarray(rate_max, np.float64)
        if len(rows) > self.CHUNK:
            return np.concatenate([self.new_period_rates(rows[i:i + self.CHUNK], cap[i:i + self.CHUNK])
                                   for i in range(0, len(rows), self.CHUNK)])
        data = self._data(rows)
        self.elas_tm1[rows], self.log_z0_tm1[rows] = self.elas_t[rows], self.log_z0_t[rows]
        elas_t, log_z0_t = self._elasticity(rows, data)
        self.elas_t[rows], self.log_z0_t[rows] = elas_t, log_z0_t
        if self.fixed_elas is not None:
            elas_t = np.full(len(rows), self.fixed_elas)
        gz, az = self._binned(data[:, :, 0])
        rates = np.clip(self._bracketize(self._bin_rates(gz, az, elas_t)), self.rate_min, cap[:, None])
        self.running_avg[rows] = self.running_avg[rows] * 0.99 + rates * 0.01
        return rates


class SaezLoop:
    """SaezBatch's interface over one SaezEstimator per replica (a Python loop): the reference's numpy calls in the
    reference's order, bit for bit.  Used for small batches - golden-trace parity runs, where a last-bit difference in a
    rate can flip a knife-edge outcome hundreds of steps later (an income of exactly zero changing sign) - while large
    batches use SaezBatch."""

    def __init__(self, n, cutoffs, rate_min, rate_max, pareto_weight_type="inverse_income", fixed_elas=None):
        self.est = [SaezEstimator(cutoffs, rate_min, rate_max, pareto_weight_type, fixed_elas) for _ in range(n)]
        self.n, self.B = int(n), self.est[0].B

    elas_tm1 = property(lambda self: np.array([e.elas_tm1 for e in self.est]))
    elas_t = property(lambda self: np.array([e.elas_t for e in self.est]))
    running_avg = property(lambda self: np.stack([e.running_avg for e in self.est]))
    count = property(lambda self: np.array([min(len(e.buffer), BUFFER_SIZE) for e in self.est]))

    def add_samples(self, rows, incomes, marginal_rates):
        for r, inc, marg in zip(rows, incomes, marginal_rates):
            self.est[int(r)].add_samples(inc, marg)

    def new_period_rates(self, rows, rate_max=None):
        caps = [None] * len(rows) if rate_max is None else list(rate_max)
        return np.stack([self.est[int(r)].new_period_rates(c) for r, c in zip(rows, caps)])


class _ReplicaView:
    """est[e]: read access to one replica's smoothed state (metrics, tests)."""

    def __init__(self, batch, e):
        self._b, self._e = batch, e

    B = property(lambda self: self._b.B)
    elas_tm1 = property(lambda self: float(self._b.elas_tm1[self._e]))
    elas_t = property(lambda self: float(self._b.elas_t[self._e]))
    running_avg = property(lambda self: self._b.running_avg[self._e])
    ready = property(lambda self: bool(self._b.count[self._e] >= BUFFER_SIZE))


class SaezHost:
    """The replica-batched estimator of a BatchedFoundationEnv plus the traffic to / from the state records."""

    EXACT_UP_TO = 64   # replicas: at or below, the per-replica loop (bit-exact restatement); above, the batched estimator

    def __init__(self, env, tax_component, estimator="auto"):
        t = tax_component
        self.env = env
        self.A = env.n_agents
        assert estimator in ("auto", "exact", "batched")
        batched = estimator == "batched" or (estimator == "auto" and env.n_envs > self.EXACT_UP_TO)
        self.batch = (SaezBatch if batched else SaezLoop)(env.n_envs, t.bracket_cutoffs, t.rate_min, t.rate_max,
                                                          t.pareto_weight_type, t.saez_fixed_elas)
        self.est = [_ReplicaView(self.batch, e) for e in range(env.n_envs)]
        # tax annealing (redistribution.py:311-330, :390-394): the maximum rate of the running episode follows the number
        # of completed episodes (components/utils.py:10-57); the formula's rates are clipped to it
        self.annealing = None if t.tax_annealing_schedule is None else (float(t._annealing_warmup), float(t._annealing_slope),
                                                                         float(t.rate_max))
        self._seen = np.zeros(env.n_envs, np.int64)   # samples already copied from the device, per replica
        self.elas_at_episode_end = [None] * env.n_envs  # saez/estimated_elasticity of previous_episode_metrics

    _SMOOTHED = ("elas_tm1", "elas_t", "log_z0_tm1", "log_z0_t")

    def state_dict(self):
        """The estimator's whole state (numpy arrays and Python values; BatchedFoundationEnv.state_dict)."""
        b = self.batch
        if isinstance(b, SaezLoop):
            out = dict(kind="loop", buffers=[np.array(e.buffer, np.float64).reshape(-1, 2) for e in b.est],
                       running_avg=np.stack([e.running_avg for e in b.est]).copy())
            out.update({k: np.array([getattr(e, k) for e in b.est], np.float64) for k in self._SMOOTHED})
        else:
            out = dict(kind="batch", buf=b.buf.copy(), count=b.count.copy(), start=b.start.copy(),
                       running_avg=b.running_avg.copy())
            out.update({k: getattr(b, k).copy() for k in self._SMOOTHED})
        out.update(seen=self._seen.copy(), elas_at_episode_end=list(self.elas_at_episode_end))
        return out

    def load_state_dict(self, sd):
        b = self.batch
        kind = "loop" if isinstance(b, SaezLoop) else "batch"
        if sd.get("kind") != kind:
            raise ValueError("load_state_dict: the Saez estimator of the checkpoint is %r, this env's is %r"
                             % (sd.get("kind"), kind))
        if kind == "loop":
            for e, est in enumerate(b.est):
                est.buffer = [[float(z), float(tau)] for z, tau in np.asarray(sd["buffers"][e], np.float64)]
                est.running_avg = np.array(sd["running_avg"][e], np.float64)
                for k in self._SMOOTHED:
                    setattr(est, k, float(sd[k][e]))
        else:
            b.buf[...], b.count[...], b.start[...] = sd["buf"], sd["count"], sd["start"]
            b.running_avg[...] = sd["running_avg"]
            for k in self._SMOOTHED:
                getattr(b, k)[...] = sd[k]
        self._seen[...] = sd["seen"]
        self.elas_at_episode_end = [None if v is None else float(v) for v in sd["elas_at_episode_end"]]

    def _np(self, name, final=False):
        st = self.env.stepper
        return st.to_numpy(st.state_view(name, final=final))

    def _write_rows(self, name, rows, values):
        """state_view(name)[rows] = values (numpy or torch backed)."""
        v = self.env.stepper.state_view(name)
        if isinstance(v, np.ndarray):
            v[rows] = values
        else:
            import torch
            v[torch.as_tensor(rows, device=v.device)] = torch.as_tensor(values, device=v.device, dtype=v.dtype)

    def before_host_reset(self):
        return self._np("saez_n").copy(), self._np("saez_rates").copy()

    def after_host_reset(self, saved):
        """An explicit env.reset() repacks the records: put the persistent Saez state back.  As in the reference
        (redistribution.py:1123 vs :1138-1139) the reset observation's curr_rates are the previous episode's last rates,
        while the rates in force become the running average."""
        saez_n, old_rates = saved
        E = self.env.n_envs
        avg = np.zeros((E, 16))
        avg[:, :self.batch.B] = self.batch.running_avg
        self._write_rows("saez_n", np.arange(E), saez_n.astype(np.int32))
        self._write_rows("saez_obs_rates", np.arange(E), old_rates)
        self._write_rows("saez_avg_rates", np.arange(E), avg)
        self._write_rows("saez_rates", np.arange(E), avg)
        if old_rates.any():
            self.env.stepper.observe()
        self.after_step()

    def after_step(self):
        """Call after every step (and after a reset): pulls new samples and, for replicas about to start a tax
        period with a full buffer, writes that period's rates."""
        n_dev = self._np("saez_n").astype(np.int64)
        t_now = self._np("t")
        fresh = np.nonzero(n_dev > self._seen)[0]
        if len(fresh):
            inc, marg = self._np("last_income")[fresh], self._np("last_marg")[fresh]
            # a replica whose episode ended on that tax day has already been reset on the device (trackers zeroed):
            # its samples are in the end-of-episode snapshot
            ended = t_now[fresh] == 0
            if ended.any():
                inc[ended] = self._np("last_income", final=True)[fresh[ended]]
                marg[ended] = self._np("last_marg", final=True)[fresh[ended]]
            self.batch.add_samples(fresh, inc, marg)   # one tax day per step at most: the A samples of the day that closed
            self._seen[fresh] = n_dev[fresh]
        for e in np.nonzero(t_now == 0)[0]:   # replicas that just finished an episode: metrics are taken before
            self.elas_at_episode_end[e] = float(self.batch.elas_tm1[e])  # the new episode's first estimate
        # replicas about to run a tax_cycle_pos == 1 step (a finished episode without auto-reset waits for its reset)
        starting = np.nonzero((self._np("tax_pos") == 1) & (n_dev >= BUFFER_SIZE) &
                              (t_now < self.env.episode_length))[0]
        if len(starting) == 0:
            return
        B = self.batch.B
        rates, avg = np.zeros((len(starting), 16)), np.zeros((len(starting), 16))
        cap = None
        if self.annealing is not None:
            warm, slope, full = self.annealing
            done = self._np("completions")[starting].astype(np.float64)
            cap = np.maximum(0.0, np.minimum(1.0, slope * (done - warm))) * full
        rates[:, :B] = self.batch.new_period_rates(starting, cap)
        avg[:, :B] = np.asarray(self.batch.running_avg)[starting]
        self._write_rows("saez_rates", starting, rates)
        self._write_rows("saez_avg_rates", starting, avg)
