"""
inference.py -- hyper-parameter inference behind `.fit()` (SURVEY.md section 8f-1).

The reference hands `ExactGP.model` (gpax/models/gp.py:137-164) to NumPyro: NUTS/MCMC for ExactGP.fit
(gp.py:207-218) and SVI with Adam(b1=0.5) and an AutoDelta / AutoNormal guide for viGP.fit (vigp.py:108-120).
Here the model's log joint is evaluated directly: the likelihood term and its gradient come from the GPU
(b2gp_mll: Cholesky + solves + fused gradient reduction), the priors are the LogNormal(0,1) defaults of
gp.py:222-247 (or gpax_b200.priors objects), and the samplers / optimiser are small host-side NumPy loops.
Custom `kernel_prior` / `noise_prior` / `mean_fn_prior` *programs* are run on the host through gpax_b200.priors'
`sample` / `plate` primitives (ProgramLogJoint); a program written against NumPyro itself cannot be interpreted here.
"""
import math

import numpy as np

from . import priors as P
from .utils import seed_from_key


def _is_nngp(kind):
    """the fused NNGP kernels (iBNN / vi_iBNN): theta = (depth [d], var_w, noise, var_b)"""
    return kind in ("NNGP_erf", "NNGP_relu")


class LogJoint:
    """log p(y, theta) over the unconstrained vector u, with gradient; theta = (k_length[d], k_scale, noise[, period]).
    Default priors and `*_prior_dist` objects only; `make_log_joint` picks ProgramLogJoint when the model carries prior
    programs (kernel_prior / noise_prior / mean_fn_prior)."""

    def __init__(self, model, jitter=1e-6):
        if model._fused is None:
            raise NotImplementedError("fit() needs kernel 'RBF', 'Matern' or 'Periodic'")
        if model.kernel_prior is not None or model.noise_prior is not None or \
                (model.mean_fn is not None and model.mean_fn_prior is not None):
            raise NotImplementedError("prior programs go through ProgramLogJoint (inference.make_log_joint)")
        self.m, self.jitter = model, float(jitter)
        X, y = model._train_arrays()
        self.X, self.d = X, X.shape[1]
        self.y = y if model.mean_fn is None else y - np.asarray(model.mean_fn(X), dtype=np.float64).squeeze()
        self.kind = model._fused
        d = self.d
        lp = model.lengthscale_prior_dist or P.LogNormal(0.0, 1.0)       # gp.py:235-239
        npd = model.noise_prior_dist or P.LogNormal(0.0, 1.0)            # gp.py:222-227
        self.names = ["k_length"] * d + ["k_scale", "noise"]
        self.priors = [lp] * d + [P.LogNormal(0.0, 1.0), npd]            # gp.py:240
        self.idx = list(range(d + 2))                                     # position in the (d+3) theta vector
        if self.kind == "Periodic":                                       # gp.py:241-244
            self.names.append("period")
            self.priors.append(P.LogNormal(0.0, 1.0))
            self.idx.append(d + 2)
        for pr in self.priors:
            if not isinstance(pr, P.Prior):
                raise TypeError("priors must be gpax_b200.priors objects (numpyro distributions cannot be used here)")
        self.dim = len(self.priors)
        self.n_evals = 0

    def theta_of(self, u):
        th = np.ones(self.d + 3)
        for k, (pr, i) in enumerate(zip(self.priors, self.idx)):
            th[i] = pr.transform(u[k])
        return th

    def init_u(self):
        """init_to_median: the reference's NUTS uses init_to_median(num_samples=10) (gp.py:208); exact medians here"""
        return np.array([float(pr.inverse(pr.median())) for pr in self.priors])

    def __call__(self, u, jacobian):
        """log p(y | theta(u)) + sum log p(theta_k) [+ log |dtheta/du| if jacobian]; returns (value, grad_u)"""
        th = self.theta_of(u)
        val, g, info = self._lik(th)
        self.n_evals += 1
        return self._joint(u, th, val, g, info, jacobian)

    @property
    def batch(self):
        """`batch(U, jacobian) -> (values [k], grads [k, dim])`: the rows of U in one b2gp_mll_draws call, row r being
        self(U[r], jacobian) bit for bit (run_nuts' vectorized chains); None for likelihoods other than b2gp_mll's"""
        return self._batch if type(self)._lik is LogJoint._lik else None

    def _batch(self, U, jacobian):
        TH = np.stack([self.theta_of(u) for u in U])
        vals, G, _, info = self.m.ctx.mll_draws(self.kind, self.X, self.y, TH, self.jitter, want_grad=True)
        self.n_evals += len(U)
        out = [self._joint(u, th, float(v), g, int(i), jacobian) for u, th, v, g, i in zip(U, TH, vals, G, info)]
        return np.array([o[0] for o in out]), np.stack([o[1] for o in out])

    def _joint(self, u, th, val, g, info, jacobian):
        """the log joint and its gradient w.r.t. u from the likelihood's value, d/dlog(theta) and info at theta(u)"""
        if info != 0 or not np.isfinite(val):
            return -np.inf, np.zeros(self.dim)
        grad = np.zeros(self.dim)
        for k, (pr, i) in enumerate(zip(self.priors, self.idx)):
            t = th[i]
            dt = float(pr.dtheta_du(u[k]))
            val += float(pr.log_prob(t))
            grad[k] = g[i] / t * dt + float(pr.dlog_prob(t)) * dt       # g is d/dlog(theta)
            if jacobian:
                val += float(pr.log_abs_jac(u[k]))
                grad[k] += float(pr.dlog_abs_jac(u[k]))
        return val, grad

    def _lik(self, th):
        """log p(y | theta) and its gradient w.r.t. log(theta): the exact marginal likelihood (b2gp_mll)"""
        val, g, _, info = self.m.ctx.mll(self.kind, self.X, self.y, th, self.jitter, want_grad=True)
        return val, g, info

    def to_dict(self, U):
        """rows of unconstrained vectors -> dict of constrained samples with the reference's site names / shapes"""
        U = np.atleast_2d(U)
        th = np.stack([self.theta_of(u) for u in U])
        out = {"k_length": th[:, :self.d], "k_scale": th[:, self.d], "noise": th[:, self.d + 1]}
        if self.kind == "Periodic":
            out["period"] = th[:, self.d + 2]
        return out


class NNGPLogJoint(LogJoint):
    """LogJoint of iBNN / vi_iBNN with their default priors (ibnn.py:54-61, vi_ibnn.py:53-60): sites var_b, var_w, noise
    in the reference's order; theta = (depth [d], var_w, noise, var_b).  The depth slots are constants: no site, no
    gradient, and nothing is divided by them."""

    def __init__(self, model, jitter=1e-6):
        if model.kernel_prior is not None or model.noise_prior is not None or \
                (model.mean_fn is not None and model.mean_fn_prior is not None):
            raise NotImplementedError("prior programs go through ProgramLogJoint (inference.make_log_joint)")
        self.m, self.jitter = model, float(jitter)
        X, y = model._train_arrays()
        self.X, self.d = X, X.shape[1]
        self.y = y if model.mean_fn is None else y - np.asarray(model.mean_fn(X), dtype=np.float64).squeeze()
        self.kind = model._fused
        d = self.d
        pb, pw = model._nngp_site_priors()
        self.names = ["var_b", "var_w", "noise"]
        self.priors = [pb, pw, model.noise_prior_dist or P.LogNormal(0.0, 1.0)]     # gp.py:222-227
        self.idx = [d + 2, d, d + 1]
        for pr in self.priors:
            if not isinstance(pr, P.Prior):
                raise TypeError("priors must be gpax_b200.priors objects (numpyro distributions cannot be used here)")
        self.dim = 3
        self.n_evals = 0

    def theta_of(self, u):
        th = super().theta_of(u)
        th[:self.d] = self.m.depth
        return th

    def to_dict(self, U):
        th = np.stack([self.theta_of(u) for u in np.atleast_2d(U)])
        return {"var_b": th[:, self.d + 2], "var_w": th[:, self.d], "noise": th[:, self.d + 1]}


def gp_model_program(m, d, kind):
    """the host side of ExactGP.model (gp.py:137-154): every statement except the likelihood.  Runs under
    priors.run_program; returns (kernel-parameter dict, noise, mean-function parameter dict or None)."""
    if m.kernel_prior is not None:
        kp = m.kernel_prior()
    elif _is_nngp(getattr(m, "_fused", None)):                         # ibnn.py:54-61, vi_ibnn.py:53-60
        kp = m._sample_kernel_params()
    else:                                                              # gp.py:229-247
        lp = m.lengthscale_prior_dist or P.LogNormal(0.0, 1.0)
        with P.plate("ard", d):
            length = P.sample("k_length", lp)
        kp = {"k_length": length, "k_scale": P.sample("k_scale", P.LogNormal(0.0, 1.0))}
        kp["period"] = P.sample("period", P.LogNormal(0.0, 1.0)) if kind == "Periodic" else None
    if m.noise_prior is not None:
        noise = m.noise_prior()
    else:                                                              # gp.py:222-227
        noise = P.sample("noise", m.noise_prior_dist or P.LogNormal(0.0, 1.0))
    mp = m.mean_fn_prior() if (m.mean_fn is not None and m.mean_fn_prior is not None) else None
    return kp, noise, mp


def prior_draws(model, rng, num_samples, d):
    """`num_samples` runs of the model's prior statements with every site drawn from its prior (what NumPyro's Predictive
    does for gp.py:401-408): list of (kernel params, noise, mean params)"""
    kind = model.kernel_name if isinstance(model.kernel_name, str) else None
    return [P.run_program(lambda: gp_model_program(model, d, kind), rng=rng)[0] for _ in range(int(num_samples))]


class ProgramLogJoint:
    """The log joint of ExactGP.model (gp.py:137-164) when some of its priors are *programs*: `kernel_prior()` returning
    the kernel-parameter dict (gp.py:141-142), the deprecated `noise_prior()` (gp.py:146-147), `mean_fn_prior()` feeding a
    parametric mean function (gp.py:151-154).  The programs are written against gpax_b200.priors' `sample` / `plate`
    (the reference's run under NumPyro).  The model program is re-run on the host for every evaluation:

      u  --transform per site-->  site values  --programs-->  theta[d+3], mean vector m[N]
      value = log N(y - m; 0, K_theta) [GPU: b2gp_mll]  +  sum_sites log p(site)  (+ log |d site / du|)

    Gradient.  The GPU returns d value / d log(theta) and alpha = K^-1 (y - m) = d value / d m.  The programs are plain
    Python (no tracer to differentiate them), so the Jacobians d theta / du and d m / du are taken by central differences
    of the host program -- 2 dim runs of a function of a handful of scalars and one [N]-vector, exact to ~1e-10 relative;
    the N^3 part is never differenced.  Site log-densities are differentiated analytically; when a program makes one
    site's distribution depend on another site's value (a hierarchical prior), the prior term's gradient is differenced
    too."""

    FD_STEP = 1e-5
    CALLABLE_KERNEL = False      # GramLogJoint: the kernel is the model's callable, not a fused GPU kernel

    def __init__(self, model, jitter=1e-6, lik=None):
        if model._fused is None and not self.CALLABLE_KERNEL:
            raise NotImplementedError("fit() needs kernel 'RBF', 'Matern' or 'Periodic'")
        self.m, self.jitter = model, float(jitter)
        X, y = model._train_arrays()
        self.X, self.d, self.y0 = X, X.shape[1], y
        self.kind = model._fused
        self.has_mean_params = model.mean_fn is not None and model.mean_fn_prior is not None
        self.fixed_mean = None
        if model.mean_fn is not None and not self.has_mean_params:
            self.fixed_mean = np.asarray(model.mean_fn(X), dtype=np.float64).squeeze()
        self._lik_fn = lik
        self._find_sites()
        self.n_evals = 0

    def _find_sites(self):
        """the model program's sites, the dimension of u, and whether any site's distribution depends on the values of
        the others (two runs at different values)"""
        _, sites, _ = P.run_program(self._model_program)
        self.sites = list(sites.values())
        self.dim = sum(s.size for s in self.sites)
        vals = {s.name: np.asarray(s.prior.transform(np.full(s.shape, 0.37))) for s in self.sites}
        _, sites2, _ = P.run_program(self._model_program, vals)
        self.hierarchical = any(vars(sites[k].prior) != vars(sites2[k].prior) for k in sites)

    def _model_program(self):
        return gp_model_program(self.m, self.d, self.kind)

    def _site_values(self, u):
        """u -> {site name: constrained value, shaped as the program sampled it}"""
        vals, o = {}, 0
        for s in self.sites:
            vals[s.name] = np.asarray(s.prior.transform(u[o:o + s.size])).reshape(s.shape)
            o += s.size
        return vals

    def _program_at(self, u):
        """u -> the model program's (kernel-parameter dict, noise, mean-function parameters) and its sites with values"""
        (kp, noise, mp), sites, _ = P.run_program(self._model_program, self._site_values(u))
        return kp, noise, mp, sites

    def _run(self, u):
        """u -> (theta[d+3], mean vector or None, sites with values)"""
        kp, noise, mp, sites = self._program_at(u)
        th = np.ones(self.d + 3)
        if _is_nngp(self.kind):
            th[:] = self.m._theta(dict(kp, noise=noise), self.d, False)[0]
            return th, self._mean(mp), sites
        th[:self.d] = np.broadcast_to(np.asarray(kp["k_length"], dtype=np.float64).reshape(-1), (self.d,)) \
            if np.size(kp["k_length"]) in (1, self.d) else np.nan
        th[self.d] = float(np.asarray(kp["k_scale"]).reshape(-1)[0])
        th[self.d + 1] = float(np.asarray(noise).reshape(-1)[0])
        if self.kind == "Periodic":
            if kp.get("period") is None:
                raise ValueError("the Periodic kernel needs 'period' in the dict kernel_prior returns")
            th[self.d + 2] = float(np.asarray(kp["period"]).reshape(-1)[0])
        return th, self._mean(mp), sites

    def _mean(self, mp):
        """the mean-function vector at X for the mean-function parameters mp, or None"""
        if self.has_mean_params:
            return np.asarray(self.m.mean_fn(self.X, mp), dtype=np.float64).squeeze()
        return self.fixed_mean

    def init_u(self):
        """init_to_median (gp.py:208)"""
        return np.concatenate([np.full(s.size, float(s.prior.inverse(s.prior.median()))) for s in self.sites])

    def _log_prior(self, u, sites, jacobian, want_grad=True):
        val, grad, o = 0.0, np.zeros(self.dim), 0
        for s0 in self.sites:
            pr = sites[s0.name].prior
            uu = u[o:o + s0.size]
            t = np.asarray(pr.transform(uu), dtype=np.float64)
            val += float(np.sum(pr.log_prob(t)))
            if want_grad:
                grad[o:o + s0.size] = np.asarray(pr.dlog_prob(t)) * np.asarray(pr.dtheta_du(uu))
            if jacobian:
                val += float(np.sum(pr.log_abs_jac(uu)))
                if want_grad:
                    grad[o:o + s0.size] += np.asarray(pr.dlog_abs_jac(uu))
            o += s0.size
        return val, grad

    def _lik(self, th, yres):
        """log p(y | theta, m) with d/dlog(theta) and alpha = K^-1 (y - m)"""
        if self._lik_fn is not None:
            return self._lik_fn(th, yres)
        val, g, alpha, info = self.m.ctx.mll(self.kind, self.X, yres, th, self.jitter, want_grad=True,
                                             want_alpha=self.has_mean_params)
        return val, g, alpha, info

    def _valid(self, th):
        if _is_nngp(self.kind):     # the depth slots may be 0; var_w, noise and var_b must be positive
            return np.all(np.isfinite(th)) and np.all(th[self.d:] > 0)
        return np.all(np.isfinite(th)) and np.all(th[:self.d + 2] > 0)

    def _dval_dth(self, th, g):
        """d value / d theta from the likelihood's gradient g, which is d/dlog(theta); unused entries carry g = 0"""
        if _is_nngp(self.kind):     # the depth slots are constants (their g is 0, and the depth may be 0)
            out = np.zeros_like(th)
            out[self.d:] = g[self.d:] / th[self.d:]
            return out
        return g / th

    def __call__(self, u, jacobian):
        u = np.asarray(u, dtype=np.float64)
        th, mean, sites = self._run(u)
        self.n_evals += 1
        if not self._valid(th):
            return -np.inf, np.zeros(self.dim)
        yres = self.y0 if mean is None else self.y0 - mean
        val, g, alpha, info = self._lik(th, yres)
        return self._joint(u, th, sites, val, g, alpha, info, jacobian)

    @property
    def batch(self):
        """`batch(U, jacobian) -> (values [k], grads [k, dim])`: the host programs and their central differences per row,
        the likelihoods of every valid row in one b2gp_mll_draws call with per-row residuals; row r is self(U[r],
        jacobian) bit for bit.  None for likelihoods other than b2gp_mll's (callable kernels, multi-task, the VFE bound)."""
        exact = type(self)._lik is ProgramLogJoint._lik and self._lik_fn is None and not self.CALLABLE_KERNEL
        return self._batch if exact and type(self).__call__ is ProgramLogJoint.__call__ else None

    def _batch(self, U, jacobian):
        rows = []
        for u in U:
            u = np.asarray(u, dtype=np.float64)
            th, mean, sites = self._run(u)
            rows.append((u, th, sites, self.y0 if mean is None else self.y0 - mean))
        self.n_evals += len(rows)
        out = [(-np.inf, np.zeros(self.dim))] * len(rows)
        live = [r for r, row in enumerate(rows) if self._valid(row[1])]
        if live:
            vals, G, A, info = self.m.ctx.mll_draws(self.kind, self.X, np.stack([rows[r][3] for r in live]),
                                                    np.stack([rows[r][1] for r in live]), self.jitter, want_grad=True,
                                                    want_alpha=self.has_mean_params)
            for j, r in enumerate(live):
                u, th, sites, _ = rows[r]
                out[r] = self._joint(u, th, sites, float(vals[j]), G[j], None if A is None else A[j], int(info[j]), jacobian)
        return np.array([o[0] for o in out]), np.stack([o[1] for o in out])

    def _joint(self, u, th, sites, val, g, alpha, info, jacobian):
        """the log joint and its gradient w.r.t. u from the likelihood at theta(u) (value, d/dlog(theta), alpha, info)"""
        if info != 0 or not np.isfinite(val):
            return -np.inf, np.zeros(self.dim)
        # site densities: analytic gradient, unless the programs are hierarchical (then differenced with the rest below)
        lp, grad = self._log_prior(u, sites, jacobian, want_grad=not self.hierarchical)
        # chain rule through the host programs by central differences
        h = self.FD_STEP
        dval_dth = self._dval_dth(th, g)
        if self.has_mean_params and alpha is None:
            raise NotImplementedError("this likelihood does not return d value / d mean: no probabilistic mean function")
        for k in range(self.dim):
            e = np.zeros(self.dim)
            e[k] = h
            thp, mp_, sp = self._run(u + e)
            thm, mm_, sm_ = self._run(u - e)
            grad[k] += float(np.dot(dval_dth, (thp - thm) / (2 * h)))
            if self.has_mean_params:
                grad[k] += float(np.dot(alpha, (mp_ - mm_) / (2 * h)))
            if self.hierarchical:
                lpp, _ = self._log_prior(u + e, sp, jacobian, want_grad=False)
                lpm, _ = self._log_prior(u - e, sm_, jacobian, want_grad=False)
                grad[k] += (lpp - lpm) / (2 * h)
        return val + lp, grad

    def to_dict(self, U):
        """rows of unconstrained vectors -> dict of constrained site values, shapes as the program sampled them"""
        U = np.atleast_2d(U)
        out = {s.name: np.empty((U.shape[0],) + s.shape) for s in self.sites}
        for r, u in enumerate(U):
            o = 0
            for s in self.sites:
                out[s.name][r] = np.asarray(s.prior.transform(u[o:o + s.size])).reshape(s.shape)
                o += s.size
        return out


class GramLogJoint(ProgramLogJoint):
    """The log joint of an ExactGP / viGP whose kernel is a user callable k(X, Z, params, noise, jitter) (gp.py:137-164
    with any kernel gpax's get_kernel passes through).  Sites are those of ProgramLogJoint: the kernel_prior program's,
    or the defaults of gp.py:229-247 over the model's kernel_dim with "period": None in the dict the callable receives.

    One evaluation at u runs the program, calls the kernel once for K = k(X, X, params, noise, jitter) and, for every
    coordinate u_k that moves the kernel dict or the noise, twice more for the central difference
    dK_k = (K(u + h e_k) - K(u - h e_k)) / 2h.  One b2gp_mll_gram call then returns the value, the traces
    d value / du_k = 1/2 sum (alpha alpha^T - K^-1) * dK_k and alpha = K^-1 (y - m): the N^3 factorisation is never
    differenced, each direction costs two N^2 kernel evaluations on the host.  Coordinates of mean_fn_prior sites get
    alpha . dm/du_k and no kernel evaluation; the prior terms are ProgramLogJoint's."""

    CALLABLE_KERNEL = True

    def __init__(self, model, jitter=1e-6):
        super().__init__(model, jitter)
        mean_sites = set()
        if self.has_mean_params:     # mean_fn_prior runs after, and apart from, the kernel and noise statements
            _, ms, _ = P.run_program(model.mean_fn_prior)
            mean_sites = set(ms)
        self.moves_kernel = np.concatenate([np.full(s.size, s.name not in mean_sites) for s in self.sites]) \
            if self.sites else np.zeros(0, dtype=bool)
        self.kernel_evals = 0

    def _model_program(self):
        return gp_model_program(self.m, self.m.kernel_dim, None)

    def _gram(self, kp, noise):
        self.kernel_evals += 1
        return np.asarray(self.m.kernel(self.X, self.X, kp, noise, jitter=self.jitter), dtype=np.float64)

    def __call__(self, u, jacobian):
        u = np.asarray(u, dtype=np.float64)
        kp, noise, mp, sites = self._program_at(u)
        self.n_evals += 1
        K = self._gram(kp, noise)
        if not np.all(np.isfinite(K)):
            return -np.inf, np.zeros(self.dim)
        mean = self._mean(mp)
        yres = self.y0 if mean is None else self.y0 - mean
        h = self.FD_STEP
        dKs, kcoords, dmean = [], [], {}
        for k in range(self.dim):
            if not (self.moves_kernel[k] or self.has_mean_params):
                continue
            e = np.zeros(self.dim)
            e[k] = h
            kpp, npl, mpp, _ = self._program_at(u + e)
            kpm, nmi, mpm, _ = self._program_at(u - e)
            if self.moves_kernel[k]:
                dKs.append((self._gram(kpp, npl) - self._gram(kpm, nmi)) / (2 * h))
                kcoords.append(k)
            if self.has_mean_params:
                dmean[k] = (self._mean(mpp) - self._mean(mpm)) / (2 * h)
        val, g, alpha, info = self.m.ctx.mll_gram(K, yres, dKs, want_grad=True, want_alpha=self.has_mean_params)
        if info != 0 or not np.isfinite(val):
            return -np.inf, np.zeros(self.dim)
        lp, grad = self._log_prior(u, sites, jacobian, want_grad=not self.hierarchical)
        grad[kcoords] += g
        for k, dm in dmean.items():
            grad[k] += float(np.dot(alpha, dm))
        if self.hierarchical:
            for k in range(self.dim):
                e = np.zeros(self.dim)
                e[k] = h
                lpp, _ = self._log_prior(u + e, self._program_at(u + e)[3], jacobian, want_grad=False)
                lpm, _ = self._log_prior(u - e, self._program_at(u - e)[3], jacobian, want_grad=False)
                grad[k] += (lpp - lpm) / (2 * h)
        return val + lp, grad


def mtgp_model_program(m, d, T, R, L):
    """the host side of MultiTaskGP.model (gpax/models/mtgp.py:92-142, 147-207): every statement except the likelihood,
    sites in the reference's order.  Returns (kernel-parameter dict, noise, mean-function parameter dict or None)."""
    if m.data_kernel_prior is not None:
        kp = dict(m.data_kernel_prior())
    else:                                                              # mtgp.py:187-207
        squeeze = (lambda x: np.squeeze(x)) if L > 1 else (lambda x: x)
        with P.plate("latent_plate_data", L, dim=-2):
            with P.plate("ard", d, dim=-1):
                length = P.sample("k_length", m.lengthscale_prior_dist or P.LogNormal(0.0, 1.0))
            if m.output_scale:
                scale = P.sample("k_scale", P.LogNormal(0.0, 1.0))
            else:
                scale = P.deterministic("k_scale", np.ones(L))
            period = P.sample("period", P.LogNormal(0.0, 1.0)) if m.data_kernel_name == "Periodic" else None
        kp = {"k_length": squeeze(length), "k_scale": squeeze(scale), "period": None if period is None else squeeze(period)}
    with P.plate("latent_plate_task", L):                              # mtgp.py:164-185
        kp["W"] = P.sample("W", m.W_prior_dist or P.Normal(0.0, 10.0).expand((L, T, R)))
        kp["v"] = P.sample("v", m.v_prior_dist or P.LogNormal(0.0, 1.0).expand((L, T)))
    if m.noise_prior is not None:
        noise = m.noise_prior()
    else:                                                              # mtgp.py:147-157
        noise = P.sample("noise", m.noise_prior_dist or P.LogNormal(0.0, 1.0).expand((T,)))
    mp = m.mean_fn_prior() if (m.mean_fn is not None and m.mean_fn_prior is not None) else None
    return kp, noise, mp


def corgp_model_program(m, d, T, R):
    """the host side of CoregGP.model (gpax/models/corgp.py:57-113 with gp.py:229-247 for the data kernel)"""
    if m.data_kernel_prior is not None:
        kp = dict(m.data_kernel_prior())
    else:
        with P.plate("ard", d):
            length = P.sample("k_length", m.lengthscale_prior_dist or P.LogNormal(0.0, 1.0))
        kp = {"k_length": length, "k_scale": P.deterministic("k_scale", np.array(1.0)),
              "period": P.sample("period", P.LogNormal(0.0, 1.0)) if m.data_kernel_name == "Periodic" else None}
    if m.task_kernel_prior is not None:
        kp.update(m.task_kernel_prior())
    else:                                                              # corgp.py:105-113
        kp["W"] = P.sample("W", P.Normal(0.0, 10.0).expand((T, R)))
        kp["v"] = P.sample("v", P.LogNormal(0.0, 1.0).expand((T,)))
    if m.noise_prior is not None:
        noise = m.noise_prior()
    else:                                                              # corgp.py:82-88
        noise = P.sample("noise", P.LogNormal(0.0, 1.0).expand((T,)))
    mp = m.mean_fn_prior() if (m.mean_fn is not None and m.mean_fn_prior is not None) else None
    return kp, noise, mp


class MTLogJoint(ProgramLogJoint):
    """ProgramLogJoint of MultiTaskGP / CoregGP: the model program yields the flat parameter vector
    p = (theta [L, d+2], B [L, T, T], noise [T]) of the LCM covariance, the GPU (b2gp_mll_multitask) returns the value,
    d value / d(log theta, B, log noise) and alpha; d p / du and d mean / du are central differences of the program, so
    custom data_kernel_prior / task_kernel_prior / noise_prior / mean_fn_prior and every *_prior_dist work unchanged."""

    def __init__(self, model, jitter=1e-6):
        self.T, self.R, self.L = model._num_tasks(), model._rank(), model._num_latents()
        super().__init__(model, jitter)
        self.rows = model._rows(self.X)
        self.nth = self.L * (model.kernel_dim + 2)

    def _model_program(self):
        return self.m._model_program(self.T, self.R, self.L)

    def _run(self, u):
        (kp, noise, mp), sites, _ = P.run_program(self._model_program, self._site_values(u))
        theta, B, nz = self.m._pack(dict(kp, noise=noise), batched=False)
        p = np.concatenate([theta.ravel(), B.ravel(), nz.ravel()])
        mean = None
        if self.has_mean_params:
            mean = np.asarray(self.m.mean_fn(self.X, mp), dtype=np.float64).squeeze()
        elif self.fixed_mean is not None:
            mean = self.fixed_mean
        return p, mean, sites

    def _split(self, p):
        nb = self.L * self.T * self.T
        return p[:self.nth], p[self.nth:self.nth + nb], p[self.nth + nb:]

    def _valid(self, p):
        th, _, nz = self._split(p)
        return np.all(np.isfinite(p)) and np.all(th > 0) and np.all(nz > 0)

    def _dval_dth(self, p, g):
        th, _, nz = self._split(p)
        gth, gB, gn = self._split(g)
        return np.concatenate([gth / th, gB, gn / nz])

    def _lik(self, p, yres):
        th, B, nz = self._split(p)
        Xd, task, group = self.rows
        val, gt, gB, gn, alpha, info = self.m.ctx.mll_multitask(
            self.m._fused, Xd, task, yres, th.reshape(self.L, -1), B.reshape(self.L, self.T, self.T), nz, group, self.jitter,
            want_grad=True, want_alpha=self.has_mean_params)
        return val, np.concatenate([gt.ravel(), gB.ravel(), gn]), alpha, info

    def to_dict(self, U):
        out = super().to_dict(U)
        if "k_scale" not in out and self.m.data_kernel_prior is None:    # numpyro.deterministic sites are in the samples
            out["k_scale"] = np.ones((np.atleast_2d(U).shape[0],) + self.m._scale_shape())
        return out


def make_log_joint(model, jitter=1e-6):
    from .gp import ExactGP
    from .vigp import viGP
    if model._fused is None and type(model) in (ExactGP, viGP):
        return GramLogJoint(model, jitter)
    if model.kernel_prior is not None or model.noise_prior is not None or \
            (model.mean_fn is not None and model.mean_fn_prior is not None):
        return ProgramLogJoint(model, jitter)
    if _is_nngp(model._fused):
        return NNGPLogJoint(model, jitter)
    return LogJoint(model, jitter)


# ---------------------------------------------------------------------------------------------- SVI
class SVIState:
    def __init__(self, losses, guide, loc, scale):
        self.losses, self.guide, self.loc, self.scale = losses, guide, loc, scale


def adam(params, objective, num_steps, step_size, progress_bar):
    """Adam(step_size, b1=0.5), the optimiser of every SVI fit here (vigp.py:108-120, sparse_gp.py:116-171,
    vidkl.py:134): maximises `objective(params) -> (elbo, grad)` and returns (params, losses = -elbo per step)."""
    m1, m2 = np.zeros_like(params), np.zeros_like(params)
    b1, b2, eps = 0.5, 0.999, 1e-8
    losses = []
    for t in range(1, int(num_steps) + 1):
        elbo, grad = objective(params)
        losses.append(-elbo)
        if not np.isfinite(elbo):
            grad = np.zeros_like(params)
        m1 = b1 * m1 + (1 - b1) * (-grad)
        m2 = b2 * m2 + (1 - b2) * grad * grad
        params = params - step_size * (m1 / (1 - b1 ** t)) / (np.sqrt(m2 / (1 - b2 ** t)) + eps)
        if progress_bar and (t % max(1, num_steps // 10) == 0 or t == num_steps):
            print(f"svi step {t}/{num_steps}  loss {losses[-1]:.4f}")
    return params, losses


def fit_vi_gp(model, rng_key, num_steps, step_size, progress_bar, **kwargs):
    """vigp.py:108-120: Adam(step_size, b1=0.5), AutoDelta (MAP in the constrained space, no Jacobian) or AutoNormal
    (mean-field normal over u, init scale 0.1, one reparameterised draw per step).  Returns (state, median dict)."""
    lj = make_log_joint(model, kwargs.get("jitter", 1e-6))
    rng = seed_from_key(rng_key)
    normal = model.guide_type == "normal"
    loc = lj.init_u()
    rho = np.full(lj.dim, math.log(0.1))            # log sigma
    params = np.concatenate([loc, rho]) if normal else loc.copy()

    def objective(params):
        if normal:
            mu, r = params[:lj.dim], params[lj.dim:]
            e = rng.standard_normal(lj.dim)
            val, g = lj(mu + np.exp(r) * e, jacobian=True)
            elbo = val + r.sum() + 0.5 * lj.dim * (1 + math.log(2 * math.pi))
            return elbo, np.concatenate([g, g * e * np.exp(r) + 1.0])
        return lj(params, jacobian=False)
    params, losses = adam(params, objective, num_steps, step_size, progress_bar)
    loc = params[:lj.dim]
    med = {k: (v[0] if v.ndim == 1 else v[0]) for k, v in lj.to_dict(loc).items()}   # guide median (vigp.py:125-127)
    return SVIState(np.array(losses), "normal" if normal else "delta", loc, np.exp(params[lj.dim:]) if normal else None), med


class SparseLogJoint(LogJoint):
    """LogJoint whose likelihood term is the VFE bound of viSparseGP.model (sparse_gp.py:62-114) at the current
    inducing inputs `self.Xu`; the gradient w.r.t. Xu of the last evaluation is left in `self.grad_Xu`."""

    def __init__(self, model, Xu, jitter=1e-6):
        super().__init__(model, jitter)
        self.Xu = np.array(Xu, dtype=np.float64, copy=True)
        if self.Xu.ndim == 1:
            self.Xu = self.Xu[:, None]
        self.grad_Xu = np.zeros_like(self.Xu)

    def _lik(self, th):
        val, g, gx, info = self.m.ctx.sparse_elbo(self.kind, self.Xu, self.X, self.y, th, self.jitter)
        self.grad_Xu = gx
        return val, g, info


def _sparse_program_log_joint(model, Xu0, jitter):
    """ProgramLogJoint over the VFE bound; carries `Xu` / `grad_Xu` like SparseLogJoint.  With a probabilistic mean
    function the device also returns alpha = (W^T W + noise I)^-1 (y - m) = d value / d m (b2gp_sparse_elbo_ex), and
    ProgramLogJoint adds alpha . dm/du_k."""
    lj = ProgramLogJoint(model, jitter, lik=None)
    lj.Xu = np.array(Xu0, dtype=np.float64, copy=True)
    if lj.Xu.ndim == 1:
        lj.Xu = lj.Xu[:, None]
    lj.grad_Xu = np.zeros_like(lj.Xu)

    def lik(th, yres):
        alpha = None
        if lj.has_mean_params:
            val, g, gx, info, alpha = model.ctx.sparse_elbo(lj.kind, lj.Xu, lj.X, yres, th, lj.jitter, want_alpha=True)
        else:
            val, g, gx, info = model.ctx.sparse_elbo(lj.kind, lj.Xu, lj.X, yres, th, lj.jitter)
        lj.grad_Xu = gx
        return val, g, alpha, info
    lj._lik_fn = lik
    return lj


def _same_params(a, b):
    """two kernel-parameter dicts hold the same values"""
    return a.keys() == b.keys() and all(
        (a[k] is None and b[k] is None) or (a[k] is not None and b[k] is not None and np.array_equal(np.asarray(a[k]), np.asarray(b[k])))
        for k in a)


class SparseGramLogJoint(GramLogJoint):
    """The log joint of viSparseGP.model (sparse_gp.py:62-114) whose kernel is a user callable k(X, Z, params, noise,
    jitter); carries `Xu` / `grad_Xu` like SparseLogJoint.  Sites are GramLogJoint's.

    One evaluation at u runs the program and makes the model's kernel calls: Kuu = k(Xu, Xu, params, jitter=jitter),
    Kuf = k(Xu, X, params) with the callable's default jitter (so with M == N its shape rule adds it, as in the
    reference), and diag(k(X, X, params, jitter=0)) from diagonal blocks of KFF_CHUNK rows (the reference forms all N x N
    entries; the diagonal is the same for a kernel that evaluates pairs independently; the blocks cost N * KFF_CHUNK
    entries, so the chunk is small).  One b2gp_sparse_elbo_gram call
    then returns the bound, its contractions with the directions below, d value / d log noise and alpha = d value / dm.

      kernel coordinates  central differences (FD_STEP) of the three blocks, as GramLogJoint;
      noise               d noise / du_k by a difference of the program (no kernel call) times the analytic derivative;
      mean_fn_prior sites alpha . dm/du_k;
      Xu                  row m of k(Xu + h e_k, Z) depends on inducing point m alone, so two shifted Kuf calls give
                          d Kuf / d Xu[:, k] for every m at once, and four shifted Kuu calls (first and second argument)
                          give rKuu_k = D1_k + D2_k^T; the row sums the library returns are grad_Xu[:, k].

    The Xu directions assume that the kernel evaluates pairs independently (k(X, Z)[i, j] depends on X[i] and Z[j]
    only): every built-in kernel and every set_kernel_fn kernel does.  The input step is XU_STEP * max(1, max |Xu[:, k]|),
    near the cube root of the fp64 epsilon that balances the O(h^2) truncation of a central difference against its
    O(eps / h) rounding."""

    KFF_CHUNK = 256
    XU_STEP = 1e-5

    def __init__(self, model, Xu, jitter=1e-6):
        super().__init__(model, jitter)
        self.Xu = np.array(Xu, dtype=np.float64, copy=True)
        if self.Xu.ndim == 1:
            self.Xu = self.Xu[:, None]
        self.grad_Xu = np.zeros_like(self.Xu)

    def _k(self, A, B, kp, **kw):
        self.kernel_evals += 1
        return np.asarray(self.m.kernel(A, B, kp, **kw), dtype=np.float64)

    def _blocks(self, kp):
        """(Kuu, Kuf, kff_diag) at the kernel parameters kp"""
        X, c = self.X, self.KFF_CHUNK
        kff = np.concatenate([np.diagonal(self._k(X[a:a + c], X[a:a + c], kp, jitter=0)) for a in range(0, X.shape[0], c)])
        return self._k(self.Xu, self.Xu, kp, jitter=self.jitter), self._k(self.Xu, X, kp), kff

    def _xu_dirs(self, kp):
        """[(rKuu_k, rKuf_k)] for every input dimension k"""
        Xu, out = self.Xu, []
        for k in range(Xu.shape[1]):
            h = self.XU_STEP * max(1.0, float(np.abs(Xu[:, k]).max()))
            e = np.zeros_like(Xu)
            e[:, k] = h
            rKuf = (self._k(Xu + e, self.X, kp) - self._k(Xu - e, self.X, kp)) / (2 * h)
            D1 = (self._k(Xu + e, Xu, kp, jitter=self.jitter) - self._k(Xu - e, Xu, kp, jitter=self.jitter)) / (2 * h)
            D2 = (self._k(Xu, Xu + e, kp, jitter=self.jitter) - self._k(Xu, Xu - e, kp, jitter=self.jitter)) / (2 * h)
            out.append((D1 + D2.T, rKuf))
        return out

    def __call__(self, u, jacobian):
        u = np.asarray(u, dtype=np.float64)
        kp, noise, mp, sites = self._program_at(u)
        self.n_evals += 1
        self.grad_Xu = np.zeros_like(self.Xu)
        noise = float(np.asarray(noise).reshape(-1)[0])
        blocks = self._blocks(kp)
        if not (noise > 0 and all(np.all(np.isfinite(b)) for b in blocks)):
            return -np.inf, np.zeros(self.dim)
        mean = self._mean(mp)
        yres = self.y0 if mean is None else self.y0 - mean
        h = self.FD_STEP
        dirs, kcoords, dnoise, dmean = [], [], np.zeros(self.dim), {}
        for k in range(self.dim):
            e = np.zeros(self.dim)
            e[k] = h
            kpp, npl, mpp, _ = self._program_at(u + e)
            kpm, nmi, mpm, _ = self._program_at(u - e)
            if not (_same_params(kpp, kp) and _same_params(kpm, kp)):
                bp, bm = self._blocks(kpp), self._blocks(kpm)
                dirs.append(tuple((p_ - m_) / (2 * h) for p_, m_ in zip(bp, bm)))
                kcoords.append(k)
            dnoise[k] = (float(np.asarray(npl).reshape(-1)[0]) - float(np.asarray(nmi).reshape(-1)[0])) / (2 * h)
            if self.has_mean_params:
                dmean[k] = (self._mean(mpp) - self._mean(mpm)) / (2 * h)
        r = self.m.ctx.sparse_elbo_gram(*blocks, yres, noise, dirs, self._xu_dirs(kp), want_alpha=self.has_mean_params)
        val = r["value"]
        if r["info"] != 0 or not np.isfinite(val):
            return -np.inf, np.zeros(self.dim)
        self.grad_Xu = r["grad_rows"].T.copy()
        lp, grad = self._log_prior(u, sites, jacobian, want_grad=not self.hierarchical)
        grad[kcoords] += r["grad"]
        grad += r["grad_log_noise"] / noise * dnoise
        for k, dm in dmean.items():
            grad[k] += float(np.dot(r["alpha"], dm))
        if self.hierarchical:
            for k in range(self.dim):
                e = np.zeros(self.dim)
                e[k] = h
                lpp, _ = self._log_prior(u + e, self._program_at(u + e)[3], jacobian, want_grad=False)
                lpm, _ = self._log_prior(u - e, self._program_at(u - e)[3], jacobian, want_grad=False)
                grad[k] += (lpp - lpm) / (2 * h)
        return val + lp, grad


def fit_sparse_gp(model, rng_key, Xu0, num_steps, step_size, progress_bar, **kwargs):
    """sparse_gp.py:116-171: SVI with Adam(b1=0.5) over the hyper-parameters (delta or normal guide, as viGP) and over
    the inducing inputs Xu (a plain parameter, no prior).  Returns (state, dict with the guide median and 'Xu')."""
    if model._fused is None:
        lj = SparseGramLogJoint(model, Xu0, kwargs.get("jitter", 1e-6))
    elif model.kernel_prior is not None or model.noise_prior is not None or \
            (model.mean_fn is not None and model.mean_fn_prior is not None):
        lj = _sparse_program_log_joint(model, Xu0, kwargs.get("jitter", 1e-6))
    else:
        lj = SparseLogJoint(model, Xu0, kwargs.get("jitter", 1e-6))
    rng = seed_from_key(rng_key)
    normal = model.guide_type == "normal"
    nu = lj.dim
    loc = lj.init_u()
    rho = np.full(nu, math.log(0.1))
    head = np.concatenate([loc, rho]) if normal else loc.copy()
    params = np.concatenate([head, lj.Xu.ravel()])
    nh = head.size

    def objective(params):
        lj.Xu = params[nh:].reshape(lj.Xu.shape)
        if normal:
            mu, r = params[:nu], params[nu:nh]
            e = rng.standard_normal(nu)
            val, g = lj(mu + np.exp(r) * e, jacobian=True)
            elbo = val + r.sum() + 0.5 * nu * (1 + math.log(2 * math.pi))
            ghead = np.concatenate([g, g * e * np.exp(r) + 1.0])
        else:
            elbo, ghead = lj(params[:nu], jacobian=False)
        return elbo, np.concatenate([ghead, lj.grad_Xu.ravel()])
    params, losses = adam(params, objective, num_steps, step_size, progress_bar)
    med = {k: v[0] for k, v in lj.to_dict(params[:nu]).items()}
    med["Xu"] = params[nh:].reshape(lj.Xu.shape)
    return SVIState(np.array(losses), "normal" if normal else "delta", params[:nu], np.exp(params[nu:nh]) if normal else None), med


# ---------------------------------------------------------------------------------------------- NUTS
class MCMCResult:
    """What ExactGP needs from numpyro's MCMC object: get_samples(group_by_chain)."""

    def __init__(self, samples_by_chain, stats):
        self._s, self.stats = samples_by_chain, stats

    def get_samples(self, group_by_chain=False):
        if group_by_chain:
            return self._s
        return {k: v.reshape((-1,) + v.shape[2:]) for k, v in self._s.items()}


# The sampler is written as generators (the *_gen functions): a chain yields each point u at which it needs the log joint and receives
# (value, grad) = lj(u, jacobian=True) back.  One implementation then serves both chain methods: "sequential" runs one
# chain's generator to its end before the next, "vectorized" advances every chain by one evaluation per round and hands
# the round's points to the log joint together.  A chain consumes its own rng in the same order either way.
def _leapfrog_gen(u, r, g, eps, minv):
    r = r + 0.5 * eps * g
    u = u + eps * minv * r
    lp, g = yield u
    r = r + 0.5 * eps * g
    return u, r, lp, g


def _find_eps_gen(u, lp, g, rng, minv):
    eps = 1.0
    r = rng.standard_normal(u.size) / np.sqrt(minv)
    h0 = lp - 0.5 * np.dot(r, minv * r)
    _, r1, lp1, _ = yield from _leapfrog_gen(u, r, g, eps, minv)
    h1 = lp1 - 0.5 * np.dot(r1, minv * r1)
    a = 1.0 if (np.isfinite(h1) and h1 - h0 > math.log(0.5)) else -1.0
    for _ in range(50):
        if not (np.isfinite(h1) and a * (h1 - h0) > -a * math.log(2)):
            if np.isfinite(h1) or a < 0:
                break
        eps *= 2.0 ** a
        _, r1, lp1, _ = yield from _leapfrog_gen(u, r, g, eps, minv)
        h1 = lp1 - 0.5 * np.dot(r1, minv * r1)
    return eps


def _nuts_draw_gen(u0, lp0, g0, eps, rng, minv, max_depth=10):
    """one transition of the no-U-turn sampler with multinomial sampling along the trajectory"""
    r0 = rng.standard_normal(u0.size) / np.sqrt(minv)
    h0 = lp0 - 0.5 * np.dot(r0, minv * r0)
    um, rm, gm = u0.copy(), r0.copy(), g0.copy()
    up, rp, gp = u0.copy(), r0.copy(), g0.copy()
    u, lp, g = u0.copy(), lp0, g0.copy()
    logw = 0.0           # log of the total weight of the current tree (relative to h0)
    depth, alpha_sum, n_alpha, diverged = 0, 0.0, 0, False

    def build(u_, r_, g_, v, j):
        nonlocal alpha_sum, n_alpha, diverged
        if j == 0:
            u1, r1, lp1, g1 = yield from _leapfrog_gen(u_, r_, g_, v * eps, minv)
            h1 = lp1 - 0.5 * np.dot(r1, minv * r1) if np.isfinite(lp1) else -np.inf
            dh = h1 - h0
            if not np.isfinite(dh):
                dh = -np.inf
            alpha_sum += min(1.0, math.exp(min(dh, 0.0))) if dh > -np.inf else 0.0
            n_alpha += 1
            ok = dh > -1000.0
            if not ok:
                diverged = True
            return u1, r1, g1, u1, r1, g1, u1, lp1, g1, dh, ok
        a = yield from build(u_, r_, g_, v, j - 1)
        um_, rm_, gm_, up_, rp_, gp_, uc, lpc, gc, lw, ok = a
        if not ok:
            return a
        if v == -1:
            b = yield from build(um_, rm_, gm_, v, j - 1)
            um_, rm_, gm_ = b[0], b[1], b[2]
        else:
            b = yield from build(up_, rp_, gp_, v, j - 1)
            up_, rp_, gp_ = b[3], b[4], b[5]
        lw2, ok2 = b[9], b[10]
        lw_tot = np.logaddexp(lw, lw2)
        if ok2 and math.log(rng.uniform()) < lw2 - lw_tot:
            uc, lpc, gc = b[6], b[7], b[8]
        span = up_ - um_
        ok = ok2 and np.dot(span, minv * rm_) >= 0 and np.dot(span, minv * rp_) >= 0     # U-turn in the metric's velocity
        return um_, rm_, gm_, up_, rp_, gp_, uc, lpc, gc, lw_tot, ok

    while depth < max_depth:
        v = 1 if rng.uniform() < 0.5 else -1
        if v == -1:
            t = yield from build(um, rm, gm, v, depth)
            um, rm, gm = t[0], t[1], t[2]
        else:
            t = yield from build(up, rp, gp, v, depth)
            up, rp, gp = t[3], t[4], t[5]
        lw2, ok = t[9], t[10]
        if ok and math.log(rng.uniform()) < lw2 - logw:      # biased progressive sampling
            u, lp, g = t[6], t[7], t[8]
        logw = np.logaddexp(logw, lw2)
        span = up - um
        if not ok or np.dot(span, minv * rm) < 0 or np.dot(span, minv * rp) < 0:
            break
        depth += 1
    return u, lp, g, alpha_sum / max(n_alpha, 1), depth, diverged


def _drive(gen, lj):
    """run a sampler generator to its end against lj(u, jacobian=True), one point at a time; returns its result"""
    try:
        u = next(gen)
        while True:
            u = gen.send(lj(u, jacobian=True))
    except StopIteration as stop:
        return stop.value


def _find_eps(lj, u, lp, g, rng, minv):
    """a reasonable first step size at u (Hoffman & Gelman, algorithm 4)"""
    return _drive(_find_eps_gen(u, lp, g, rng, minv), lj)


def _nuts_draw(lj, u0, lp0, g0, eps, rng, minv, max_depth=10):
    """one NUTS transition from u0: (u, lp, grad, mean acceptance, depth, diverged)"""
    return _drive(_nuts_draw_gen(u0, lp0, g0, eps, rng, minv, max_depth), lj)


def _chain(lj, c, seed, num_warmup, num_samples, progress_bar):
    """one NUTS chain as a generator (see _leapfrog_gen); returns (draws [num_samples, dim], step size, divergences)"""
    rng = np.random.default_rng(seed)
    u = lj.init_u() + (0.0 if c == 0 else 0.1 * rng.standard_normal(lj.dim))
    lp, g = yield u
    minv = np.ones(lj.dim)
    eps = yield from _find_eps_gen(u, lp, g, rng, minv)
    mu, hbar, log_eps_bar, gamma, t0, kappa, delta = math.log(10 * eps), 0.0, 0.0, 0.05, 10.0, 0.75, 0.8
    draws, warm_buf, div, m = [], [], 0, 0
    metric_at = (3 * int(num_warmup)) // 4 if num_warmup >= 40 else -1
    for it in range(int(num_warmup) + int(num_samples)):
        u, lp, g, acc, depth, dv = yield from _nuts_draw_gen(u, lp, g, eps, rng, minv)
        if it < num_warmup:
            m += 1
            hbar = (1 - 1 / (m + t0)) * hbar + (delta - acc) / (m + t0)
            log_eps = mu - math.sqrt(m) / gamma * hbar
            eta = m ** (-kappa)
            log_eps_bar = eta * log_eps + (1 - eta) * log_eps_bar
            eps = math.exp(log_eps)
            if num_warmup // 4 <= it < metric_at:
                warm_buf.append(u.copy())
            if it == metric_at - 1 and len(warm_buf) >= 10:
                var = np.var(np.array(warm_buf), axis=0)
                minv = (len(warm_buf) * var + 1e-3 * 5) / (len(warm_buf) + 5)        # regularised, as Stan
                eps = yield from _find_eps_gen(u, lp, g, rng, minv)                       # step size for the new metric
                mu, hbar, log_eps_bar, m = math.log(10 * eps), 0.0, 0.0, 0            # dual averaging restarts
            if it == num_warmup - 1:
                eps = math.exp(log_eps_bar) if m > 0 else eps
        else:
            draws.append(u.copy())
            div += int(dv)
        if progress_bar and (it + 1) % max(1, (num_warmup + num_samples) // 10) == 0:
            print(f"chain {c} iter {it + 1}/{num_warmup + num_samples} step {eps:.3g} depth {depth} lp {lp:.3f}")
    return np.array(draws), eps, div


def fit_exact_gp(model, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method="sequential", **kwargs):
    """gp.py:207-218."""
    return run_nuts(make_log_joint(model, kwargs.get("jitter", 1e-6)), rng_key, num_warmup, num_samples, num_chains, progress_bar,
                    chain_method=chain_method)


def run_nuts(lj, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method="sequential"):
    """NUTS over any log joint `lj(u, jacobian) -> (value, grad)` with `dim`, `init_u()`, `to_dict(U)`.  Dual-averaging
    step-size adaptation (target accept 0.8).  Warm-up windows as in Stan / NumPyro: draws of the middle of warm-up
    estimate a diagonal mass matrix, which is installed at 3/4 of warm-up; the step size is then re-initialised for the
    new metric and dual averaging restarts over the last quarter.

    chain_method "vectorized" runs the chains in lock-step: each round evaluates the pending point of every unfinished
    chain, with one `lj.batch(U, jacobian) -> (values [k], grads [k, dim])` call when the log joint has one, else row by
    row.  Every other value ("sequential", the default, and "parallel") runs the chains one after another.  Either way
    chain c draws from the same seed in the same order, so both give the same samples bit for bit as long as `batch`
    returns what `lj` returns row by row; stats[c]["grad_evals"] counts the evaluations of chains 0..c."""
    root = seed_from_key(rng_key)
    seeds = [root.integers(0, 2 ** 63) for _ in range(int(num_chains))]
    gens = [_chain(lj, c, seed, num_warmup, num_samples, progress_bar) for c, seed in enumerate(seeds)]
    n0 = lj.n_evals
    results, evals = [None] * len(gens), [0] * len(gens)
    if chain_method == "vectorized":
        batch = getattr(lj, "batch", None)
        pending = {}
        for c, gen in enumerate(gens):
            pending[c] = next(gen)
        while pending:
            cs = sorted(pending)
            if batch is not None:
                vals, grads = batch(np.stack([pending[c] for c in cs]), jacobian=True)
                outs = [(vals[i], grads[i]) for i in range(len(cs))]
                for c in cs:
                    evals[c] += 1
            else:
                outs = []
                for c in cs:
                    before = lj.n_evals
                    outs.append(lj(pending[c], jacobian=True))
                    evals[c] += lj.n_evals - before
            for c, out in zip(cs, outs):
                try:
                    pending[c] = gens[c].send(out)
                except StopIteration as stop:
                    results[c] = stop.value
                    del pending[c]
    else:
        for c, gen in enumerate(gens):
            before = lj.n_evals
            results[c] = _drive(gen, lj)
            evals[c] = lj.n_evals - before
    chains, stats, total = [], [], n0
    for (draws, eps, div), e in zip(results, evals):
        total += e
        chains.append(draws)
        stats.append({"step_size": eps, "divergences": div, "grad_evals": total})
    per_chain = [lj.to_dict(ch) for ch in chains]
    by_chain = {k: np.stack([pc[k] for pc in per_chain]) for k in per_chain[0]}
    return MCMCResult(by_chain, stats)
