"""
variants.py -- the exact-GP model variants of SURVEY.md section 8f-3 on the same C-ABI boundary:

  MeasuredNoiseGP   gpax/models/mngp.py    measured per-point noise in the likelihood (k + diag(noise), :92-97), noise
                                           extrapolated to new points at predict time (:159-247)
  VarNoiseGP        gpax/models/hskgp.py   heteroskedastic GP: a second (noise) GP over log-variances (:105-206)
  vExactGP          gpax/models/vgp.py     vector-valued targets: an outer task axis over X, y and the parameters (:55-196)
  UIGP              gpax/models/uigp.py    uncertain inputs: the training inputs X_prime are a sampled site (:78-150)

Every posterior is one b2gp_posterior_batch call (per-member inputs, per-point noise vectors); likelihoods with a
noise vector are b2gp_mll_v; the task-batched likelihood of vExactGP and UIGP's likelihood with its input gradient are
b2gp_mll_batch; samples from covariances modified on the way are b2gp_mvn_sample.  Nothing numerical runs
on the host except elementwise glue the reference also does in Python (exp of a predicted log-variance, broadcasting).
"""
import math
import warnings
from typing import Callable, Dict, Optional, Tuple

import numpy as np

from . import priors as P
from . import prng
from .gp import ExactGP, _eps_dtype, _theta_rows
from .kernels import builtin_name, get_kernel
from .utils import posterior_eps

__all__ = ["MeasuredNoiseGP", "VarNoiseGP", "vExactGP", "UIGP"]


def _need_fused(model):
    if model._fused is None:
        raise NotImplementedError("this model variant needs kernel 'RBF', 'Matern' or 'Periodic'")


# ---------------------------------------------------------------------------------------------- MeasuredNoiseGP
class _MeasuredNoiseLogJoint:
    """log joint of MeasuredNoiseGP.model (mngp.py:75-97): kernel parameters only, noise fixed at 0, likelihood
    N(y; 0, k + diag(measured_noise)) evaluated with its gradient on the GPU (b2gp_mll_v)."""

    def __init__(self, model, measured_noise, jitter):
        from .inference import LogJoint
        base = LogJoint(model, jitter)
        self.base, self.nv = base, np.asarray(measured_noise, dtype=np.float64).reshape(-1)
        keep = [k for k, nm in enumerate(base.names) if nm != "noise"]
        self.priors = [base.priors[k] for k in keep]
        self.idx = [base.idx[k] for k in keep]
        self.dim, self.d, self.kind = len(keep), base.d, base.kind
        self.n_evals = 0

    def theta_of(self, u):
        th = np.ones(self.d + 3)
        th[self.d + 1] = 0.0                                        # numpyro.deterministic("noise", 0.0), mngp.py:85
        for k, (pr, i) in enumerate(zip(self.priors, self.idx)):
            th[i] = pr.transform(u[k])
        return th

    def init_u(self):
        return np.array([float(pr.inverse(pr.median())) for pr in self.priors])

    def __call__(self, u, jacobian):
        th = self.theta_of(u)
        val, g, _, info, _ = self.base.m.ctx.mll(self.kind, self.base.X, self.base.y, th, self.base.jitter, True, False, self.nv)
        self.n_evals += 1
        return self._joint(u, th, val, g, info, jacobian)

    def batch(self, U, jacobian):
        """the rows of U (one per chain of a vectorized NUTS round) in one b2gp_mll_draws_v call with the shared measured
        noise; row r is self(U[r], jacobian) bit for bit"""
        TH = np.stack([self.theta_of(u) for u in U])
        vals, G, _, _, info = self.base.m.ctx.mll_draws_v(self.kind, self.base.X, self.base.y, TH, self.nv, self.base.jitter,
                                                          want_grad=True)
        self.n_evals += len(U)
        out = [self._joint(u, th, float(v), g, int(i), jacobian) for u, th, v, g, i in zip(U, TH, vals, G, info)]
        return np.array([o[0] for o in out]), np.stack([o[1] for o in out])

    def _joint(self, u, th, val, g, info, jacobian):
        if info != 0 or not np.isfinite(val):
            return -np.inf, np.zeros(self.dim)
        grad = np.zeros(self.dim)
        for k, (pr, i) in enumerate(zip(self.priors, self.idx)):
            t, dt = th[i], float(pr.dtheta_du(u[k]))
            val += float(pr.log_prob(t))
            grad[k] = g[i] / t * dt + float(pr.dlog_prob(t)) * dt
            if jacobian:
                val += float(pr.log_abs_jac(u[k]))
                grad[k] += float(pr.dlog_abs_jac(u[k]))
        return val, grad

    def to_dict(self, U):
        U = np.atleast_2d(U)
        th = np.stack([self.theta_of(u) for u in U])
        out = {"k_length": th[:, :self.d], "k_scale": th[:, self.d], "noise": th[:, self.d + 1]}
        if self.kind == "Periodic":
            out["period"] = th[:, self.d + 2]
        return out


class MeasuredNoiseGP(ExactGP):
    """Gaussian process with measured noise -- gpax/models/mngp.py:28-73."""

    def __init__(self, input_dim: int, kernel, mean_fn: Optional[Callable] = None, kernel_prior: Optional[Callable] = None,
                 mean_fn_prior: Optional[Callable] = None, lengthscale_prior_dist=None, ctx=None) -> None:
        super().__init__(input_dim, kernel, mean_fn, kernel_prior, mean_fn_prior, None, None, lengthscale_prior_dist, ctx=ctx)
        self.measured_noise = None
        self.noise_predicted = None

    def fit(self, rng_key, X, y, measured_noise, num_warmup: int = 2000, num_samples: int = 2000, num_chains: int = 1,
            chain_method: str = "sequential", progress_bar: bool = True, print_summary: bool = True, device=None,
            **kwargs: float) -> None:
        """mngp.py:100-158.  kernel_prior / mean_fn_prior programs go through ProgramLogJoint with the measured noise as
        its fixed noise vector."""
        from .inference import ProgramLogJoint, run_nuts
        X, y = self._set_data(X, y)
        self.X_train, self.y_train = X, y
        self.measured_noise = np.asarray(measured_noise, dtype=np.float64)
        jitter = kwargs.get("jitter", 1e-6)
        if self.kernel_prior is not None or (self.mean_fn is not None and self.mean_fn_prior is not None):
            _need_fused(self)
            lj = ProgramLogJoint(self, jitter, noise_vec=self.measured_noise)
        else:
            lj = _MeasuredNoiseLogJoint(self, self.measured_noise, jitter)
        self.mcmc = run_nuts(lj, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method)
        if print_summary:
            self._print_summary()

    def linreg(self, x, y, x_new, **kwargs):
        """mngp.py:249-252.  The reference fits alpha + x beta by SVI with wide Normal(0, 10) priors and reads the guide's
        median; with N >> d + 1 that is the least-squares line, which is what is solved here (a (d+1)-parameter problem)."""
        x, x_new = np.asarray(x, dtype=np.float64), np.asarray(x_new, dtype=np.float64)
        A = np.column_stack([np.ones(len(x)), x])
        coef, *_ = np.linalg.lstsq(A, np.asarray(y, dtype=np.float64), rcond=None)
        return coef[0] + x_new @ coef[1:]

    def gpreg(self, x, y, x_new, **kwargs):
        """mngp.py:254-258: a viGP with an RBF kernel over the measured noise."""
        from .vigp import viGP
        vigp = viGP(self.kernel_dim, "RBF", ctx=self._ctx)
        vigp.fit(0, x, y, progress_bar=False, print_summary=False, **kwargs)
        return vigp.predict(1, x_new, noiseless=True)[0]

    def predict(self, rng_key, X_new, samples: Optional[Dict[str, np.ndarray]] = None, n: int = 1, filter_nans: bool = False,
                noiseless: bool = True, device=None, noise_prediction_method: str = "linreg",
                **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """mngp.py:186-247.  Per draw (mngp.py:159-184): (mean, K) = get_mvn_posterior, K += diag(noise_predicted),
        y = mean + sqrt(clip(diag K, 0)) * normal -- only the diagonal of K is ever used, so the posterior call asks for
        the diagonal-variance epilogue and the P x P covariance is never formed."""
        _need_fused(self)
        if noise_prediction_method not in ["linreg", "gpreg"]:
            raise NotImplementedError("For noise prediction method, select between 'linreg' and 'gpreg'")
        X_new = self._set_data(X_new)
        if self.noise_predicted is not None:
            noise_predicted = self.noise_predicted
        else:
            fn = self.linreg if noise_prediction_method == "linreg" else self.gpreg
            noise_predicted = np.asarray(fn(np.asarray(self.X_train), self.measured_noise, X_new, **kwargs))
            self.noise_predicted = noise_predicted
        if samples is None:
            samples = self.get_samples(chain_dim=False)
        S = len(next(iter(samples.values())))
        out = self._posterior_batched(X_new, samples, True, noiseless, ("mean", "var"), **kwargs)
        y_means, var = out["mean"], out["var"] + noise_predicted[None, :]
        sig = np.sqrt(np.clip(var, 0.0, None))
        Pn = X_new.shape[0]
        keys = prng.split(prng.as_key(rng_key), S)                      # one key per draw (mngp.py:239)
        z = np.stack([np.stack([prng.normal(k2, (Pn,), _eps_dtype()) for k2 in prng.split(k, n)]) for k in keys])
        y_sampled = y_means[:, None, :] + sig[:, None, :] * z.astype(np.float64)
        if filter_nans:
            y_sampled = y_sampled[[i for i in range(S) if not np.isnan(y_sampled[i]).any()]]
        return y_means.mean(0), y_sampled


# ---------------------------------------------------------------------------------------------- VarNoiseGP
class VarNoiseGP(ExactGP):
    """Heteroskedastic GP -- gpax/models/hskgp.py:24-103."""

    def __init__(self, input_dim: int, kernel, noise_kernel="RBF", mean_fn: Optional[Callable] = None,
                 kernel_prior: Optional[Callable] = None, mean_fn_prior: Optional[Callable] = None,
                 noise_kernel_prior: Optional[Callable] = None, lengthscale_prior_dist=None,
                 noise_mean_fn: Optional[Callable] = None, noise_mean_fn_prior: Optional[Callable] = None,
                 noise_lengthscale_prior_dist=None, ctx=None) -> None:
        super().__init__(input_dim, kernel, mean_fn, kernel_prior, mean_fn_prior, None, None, lengthscale_prior_dist, ctx=ctx)
        self._noise_fused = builtin_name(noise_kernel)
        self.noise_kernel = get_kernel(noise_kernel)
        self.noise_mean_fn = noise_mean_fn
        self.noise_mean_fn_prior = noise_mean_fn_prior
        self.noise_kernel_prior = noise_kernel_prior
        self.noise_lengthscale_prior_dist = noise_lengthscale_prior_dist

    def _noise_theta(self, params, batched):
        """the noise kernel reads the sites k_noise_length / k_noise_scale (hskgp.py:151-163 via utils._set_noise_kernel_fn)"""
        d = self.kernel_dim
        n = {"k_length": params["k_noise_length"], "k_scale": params["k_noise_scale"],
             "noise": np.zeros_like(np.asarray(params["k_noise_scale"], dtype=np.float64)), "period": params.get("period")}
        return _theta_rows(n, d, batched)

    def _log_noise_mean(self, X, params, batched, S):
        """log noise_mean_fn at X (hskgp.py:117-121, 192-200): [N], or [S, N] when the function has a prior and params
        carry a draw axis (evaluated once per draw, as _residuals does for mean_fn)"""
        f = self.noise_mean_fn
        if self.noise_mean_fn_prior is None:
            return np.log(np.asarray(f(X), dtype=np.float64)).squeeze()
        if not batched:
            return np.log(np.asarray(f(X, params), dtype=np.float64)).squeeze()
        return np.stack([np.log(np.asarray(f(X, {k: np.asarray(v)[s] for k, v in params.items()}), dtype=np.float64)).reshape(-1)
                         for s in range(S)])

    def _both_posteriors(self, X_new, params, batched, want, **kwargs):
        """hskgp.py:165-204 for one or S draws: the main GP with ZERO noise in k_XX and k_pp, and the noise GP's
        posterior mean of the log-variances; returns (out dict of the main GP, predicted noise variance [S, P])."""
        _need_fused(self)
        if self._noise_fused is None:
            raise NotImplementedError("noise_kernel must be 'RBF', 'Matern' or 'Periodic'")
        X, y = self._train_arrays()
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        jitter = float(kwargs.get("jitter", 1e-6))
        main = dict(params)
        main["noise"] = np.zeros_like(np.asarray(params["k_scale"], dtype=np.float64))       # kernel(..., 0, **kwargs)
        theta = _theta_rows(main, X.shape[1], batched)
        S = theta.shape[0]
        yres = self._residuals(X, y, params, batched, S)
        out = self.ctx.posterior(self._fused, X, yres, Xn, theta, True, jitter, want)
        pm = self._prior_mean(Xn, params, batched, S)
        if pm is not None:
            out["mean"] = out["mean"] + pm
        log_var = np.asarray(params["log_var"], dtype=np.float64).reshape(S, -1)
        shift_tr = shift_new = 0.0
        if self.noise_mean_fn is not None:                                                    # hskgp.py:192-200
            shift_tr, shift_new = self._log_noise_mean(X, params, batched, S), self._log_noise_mean(Xn, params, batched, S)
        nout = self.ctx.posterior(self._noise_fused, X, log_var - shift_tr, Xn, self._noise_theta(params, batched), True, jitter,
                                  ("mean",))
        bad = (out["info"] != 0) | (nout["info"] != 0)
        pred_var = np.exp(nout["mean"] + shift_new)
        pred_var[bad] = np.nan
        return out, pred_var

    def get_mvn_posterior(self, X_new, params: Dict[str, np.ndarray], *args, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """hskgp.py:165-204: mean of the main GP, covariance = main GP's + diag(exp(predicted log-variance))."""
        out, pv = self._both_posteriors(X_new, params, False, ("mean", "cov"), **kwargs)
        cov = out["cov"][0]
        cov[np.diag_indices_from(cov)] += pv[0]
        return out["mean"][0], cov

    def predict(self, rng_key, X_new, samples: Optional[Dict[str, np.ndarray]] = None, n: int = 1, filter_nans: bool = False,
                noiseless: bool = False, device=None, **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """ExactGP.predict (gp.py:351-399) over this class's get_mvn_posterior: all S draws in two batched posterior calls,
        the noise variance added on the diagonal, then the sampling Cholesky of each modified covariance on the GPU."""
        X_new = self._set_data(X_new)
        if samples is None:
            samples = self.get_samples(chain_dim=False)
        S = len(next(iter(samples.values())))
        Pn = X_new.shape[0]
        out, pv = self._both_posteriors(X_new, samples, True, ("mean", "cov"), **kwargs)
        cov = out["cov"]
        idx = np.arange(Pn)
        cov[:, idx, idx] += pv
        eps = posterior_eps(rng_key, S, n, Pn, _eps_dtype())
        y_sampled, _ = self.ctx.mvn_sample(out["mean"], cov, eps)
        if filter_nans:
            y_sampled = y_sampled[[i for i in range(S) if not np.isnan(y_sampled[i]).any()]]
        return out["mean"].mean(0), y_sampled

    def get_data_var_samples(self):
        """hskgp.py:208-218."""
        samples = self.mcmc.get_samples()
        log_var = np.array(samples["log_var"], dtype=np.float64)
        if self.noise_mean_fn is not None:
            X = np.asarray(self.X_train).squeeze()
            if self.noise_mean_fn_prior is not None:
                S = log_var.shape[0]
                mean_ = np.stack([self.noise_mean_fn(X, {k: np.asarray(v)[s] for k, v in samples.items()}) for s in range(S)])
            else:
                mean_ = self.noise_mean_fn(X)
            log_var = log_var + np.log(mean_)
        return np.exp(log_var)

    def fit(self, rng_key, X, y, num_warmup: int = 2000, num_samples: int = 2000, num_chains: int = 1,
            chain_method: str = "sequential", progress_bar: bool = True, print_summary: bool = True, device=None,
            **kwargs: float) -> None:
        """NUTS over (main kernel, noise kernel, log_var[N]) for hskgp.py:105-149; both multivariate-normal terms and
        their gradients (w.r.t. the kernel parameters AND the latent log-variances) come from b2gp_mll / b2gp_mll_v.
        kernel_prior, noise_kernel_prior, mean_fn_prior and noise_mean_fn_prior programs go through
        _VarNoiseProgramLogJoint."""
        from .inference import run_nuts
        X, y = self._set_data(X, y)
        self.X_train, self.y_train = X, y
        jitter = kwargs.get("jitter", 1e-6)
        programs = self.kernel_prior is not None or self.noise_kernel_prior is not None or \
            (self.mean_fn is not None and self.mean_fn_prior is not None) or \
            (self.noise_mean_fn is not None and self.noise_mean_fn_prior is not None)
        lj = _VarNoiseProgramLogJoint(self, jitter) if programs else _VarNoiseLogJoint(self, jitter)
        self.mcmc = run_nuts(lj, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method)
        if print_summary:
            s = self.get_samples(1)
            for k, v in s.items():
                if "log_var" not in k:                                                        # hskgp.py:220-222
                    print(f"{k:>16s}  mean {np.mean(v, axis=(0, 1))}  std {np.std(v, axis=(0, 1))}")


class _VarNoiseLogJoint:
    """u = [log k_length (d), log k_scale, log k_noise_length (1), log k_noise_scale, log_var (N)] -- hskgp.py:105-163 with
    the default LogNormal(0, 1) priors (or gpax_b200.priors objects for the two lengthscales), a fixed mean_fn and a
    fixed noise_mean_fn (log_var ~ N(log noise_mean_fn(X), k_noise))."""

    def __init__(self, model, jitter):
        _need_fused(model)
        self.m, self.jitter = model, float(jitter)
        self.X, self.y = model._train_arrays()
        if model.mean_fn is not None:
            self.y = self.y - np.asarray(model.mean_fn(self.X), dtype=np.float64).squeeze()
        self.mu_n = None
        if model.noise_mean_fn is not None:
            with np.errstate(divide="ignore", invalid="ignore"):
                self.mu_n = model._log_noise_mean(self.X, None, False, 1)
        self.N, self.d = self.X.shape
        d = self.d
        lp = model.lengthscale_prior_dist or P.LogNormal(0.0, 1.0)
        nlp = model.noise_lengthscale_prior_dist or P.LogNormal(0.0, 1.0)
        self.priors = [lp] * d + [P.LogNormal(0.0, 1.0), nlp, P.LogNormal(0.0, 1.0)]
        self.nk = d + 3
        self.dim = self.nk + self.N
        self.n_evals = 0

    def init_u(self):
        u = np.zeros(self.dim)
        u[:self.nk] = [float(pr.inverse(pr.median())) for pr in self.priors]
        u[self.nk:] = np.log(0.1 * np.var(self.y) + 1e-8)
        return u

    def _thetas(self, u):
        d = self.d
        t = np.array([pr.transform(v) for pr, v in zip(self.priors, u[:self.nk])], dtype=np.float64)
        th = np.ones(d + 3)
        th[:d], th[d], th[d + 1] = t[:d], t[d], 0.0
        thn = np.ones(d + 3)
        thn[:d], thn[d], thn[d + 1] = t[d + 1], t[d + 2], 0.0
        return t, th, thn

    def _lv_res(self, lv):
        return lv if self.mu_n is None else lv - self.mu_n

    def __call__(self, u, jacobian):
        ctx = self.m.ctx
        t, th, thn = self._thetas(u)
        lv = u[self.nk:]
        self.n_evals += 1
        if self.mu_n is not None and not np.all(np.isfinite(self.mu_n)):
            return -np.inf, np.zeros(self.dim)
        vA, gA, alphaA, infoA = ctx.mll(self.m._noise_fused, self.X, self._lv_res(lv), thn, self.jitter, True, True)   # log N(log_var; mu_n, k_noise)
        vB, gB, _, infoB, gnv = ctx.mll(self.m._fused, self.X, self.y, th, self.jitter, True, False, np.exp(lv))
        return self._joint(u, t, vA, gA, alphaA, infoA, vB, gB, infoB, gnv, jacobian)

    def batch(self, U, jacobian):
        """the rows of U (one per chain of a vectorized NUTS round): one b2gp_mll_draws call for the noise GP and one
        b2gp_mll_draws_v call for the main GP; row r is self(U[r], jacobian) bit for bit"""
        ctx, U = self.m.ctx, np.asarray(U, dtype=np.float64)
        self.n_evals += len(U)
        if self.mu_n is not None and not np.all(np.isfinite(self.mu_n)):
            return np.full(len(U), -np.inf), np.zeros((len(U), self.dim))
        parts = [self._thetas(u) for u in U]
        LV = U[:, self.nk:]
        vA, GA, AA, iA = ctx.mll_draws(self.m._noise_fused, self.X, self._lv_res(LV), np.stack([p[2] for p in parts]), self.jitter,
                                       want_grad=True, want_alpha=True)
        vB, GB, _, GNV, iB = ctx.mll_draws_v(self.m._fused, self.X, self.y, np.stack([p[1] for p in parts]),
                                             np.stack([np.exp(lv) for lv in LV]), self.jitter, want_grad=True)
        out = [self._joint(u, p[0], float(vA[r]), GA[r], AA[r], int(iA[r]), float(vB[r]), GB[r], int(iB[r]), GNV[r], jacobian)
               for r, (u, p) in enumerate(zip(U, parts))]
        return np.array([o[0] for o in out]), np.stack([o[1] for o in out])

    def _joint(self, u, t, vA, gA, alphaA, infoA, vB, gB, infoB, gnv, jacobian):
        d = self.d
        lv = u[self.nk:]
        if infoA != 0 or infoB != 0 or not (np.isfinite(vA) and np.isfinite(vB)):
            return -np.inf, np.zeros(self.dim)
        val = vA + vB
        grad = np.zeros(self.dim)
        gk = np.concatenate([gB[:d], [gB[d]], [gA[:d].sum()], [gA[d]]])          # d/dlog of each sampled kernel parameter
        for k, pr in enumerate(self.priors):
            dt = float(pr.dtheta_du(u[k]))
            val += float(pr.log_prob(t[k]))
            grad[k] = gk[k] / t[k] * dt + float(pr.dlog_prob(t[k])) * dt
            if jacobian:
                val += float(pr.log_abs_jac(u[k]))
                grad[k] += float(pr.dlog_abs_jac(u[k]))
        grad[self.nk:] = -alphaA + gnv * np.exp(lv)
        return val, grad

    def to_dict(self, U):
        U = np.atleast_2d(U)
        d = self.d
        T = np.stack([self._thetas(u)[0] for u in U])
        return {"k_length": T[:, :d], "k_scale": T[:, d], "k_noise_length": T[:, d + 1:d + 2], "k_noise_scale": T[:, d + 2],
                "log_var": U[:, self.nk:], "noise": np.zeros(len(U))}


class _VarNoiseProgramLogJoint:
    """The log joint of VarNoiseGP.model (hskgp.py:105-149) when any of kernel_prior, noise_kernel_prior, mean_fn_prior,
    noise_mean_fn_prior is a program (gpax_b200.priors' sample / plate).  u holds the sites in the reference's order:
    noise-kernel sites, noise-mean sites, log_var [N], kernel sites (period for a Periodic kernel), mean sites.

      value = log N(lv; mu_n, K_n) [b2gp_mll]  +  log N(y - m; 0, K + diag(e^lv)) [b2gp_mll_v]  +  sum log p(site) (+ Jac.)

    d value / d lv = -alpha_n + g_nv e^lv in closed form.  The programs are differenced centrally over their own sites
    only (never over the N log_var coordinates): theta, theta_n, mu_n (against +alpha_n) and m (against alpha_m)."""

    FD_STEP = 1e-5
    INIT_TRIES = 100

    def __init__(self, model, jitter):
        _need_fused(model)
        if model._noise_fused is None:
            raise NotImplementedError("noise_kernel must be 'RBF', 'Matern' or 'Periodic'")
        self.m, self.jitter = model, float(jitter)
        self.kind, self.nkind = model._fused, model._noise_fused
        self.X, self.y0 = model._train_arrays()
        self.N, self.d = self.X.shape
        self.mean_params = model.mean_fn is not None and model.mean_fn_prior is not None
        self.noise_mean_params = model.noise_mean_fn is not None and model.noise_mean_fn_prior is not None
        self.fixed_mean = None if model.mean_fn is None or self.mean_params else \
            np.asarray(model.mean_fn(self.X), dtype=np.float64).squeeze()
        self.fixed_mu_n = None
        if model.noise_mean_fn is not None and not self.noise_mean_params:
            with np.errstate(divide="ignore", invalid="ignore"):
                self.fixed_mu_n = model._log_noise_mean(self.X, None, False, 1)
        _, s1, _ = P.run_program(self._noise_program)
        _, s2, _ = P.run_program(self._main_program)
        self.pre, self.post = list(s1.values()), list(s2.values())
        n1 = sum(s.size for s in self.pre)
        self.lv = slice(n1, n1 + self.N)
        self.dim = n1 + self.N + sum(s.size for s in self.post)
        # (site, its slice of u) in u's order
        self.blocks, o = [], 0
        for s in self.pre + [None] + self.post:
            if s is None:
                o += self.N
                continue
            self.blocks.append((s, slice(o, o + s.size)))
            o += s.size
        self.prog_idx = np.concatenate([np.arange(self.dim)[sl] for _, sl in self.blocks]) if self.blocks else np.zeros(0, int)
        # does any site's distribution depend on the value of another (two runs at different values)?
        sites1 = self._run(np.full(self.dim, 0.37))[4]
        self.hierarchical = any(vars(sites1[s.name].prior) != vars(s.prior) for s, _ in self.blocks)
        self._u0 = None
        self.n_evals = 0

    # ---- the host programs
    def _noise_program(self):
        m = self.m
        if m.noise_kernel_prior is not None:
            nkp = m.noise_kernel_prior()
        else:                                                                                # hskgp.py:151-163
            nkp = {"k_noise_scale": P.sample("k_noise_scale", P.LogNormal(0.0, 1.0)),
                   "k_noise_length": P.sample("k_noise_length", m.noise_lengthscale_prior_dist or P.LogNormal(0.0, 1.0))}
        nmp = m.noise_mean_fn_prior() if self.noise_mean_params else None
        return nkp, nmp

    def _main_program(self):
        from .inference import kernel_program
        kp = kernel_program(self.m, self.d, self.kind)
        mp = self.m.mean_fn_prior() if self.mean_params else None
        return kp, mp

    def _run(self, u):
        """u -> (theta [d+3], theta_n [d+3], m [N] or None, mu_n [N] or None, sites with their priors)"""
        vals = {s.name: np.asarray(s.prior.transform(u[sl])).reshape(s.shape) for s, sl in self.blocks}
        (nkp, nmp), s1, _ = P.run_program(self._noise_program, vals)
        (kp, mp), s2, _ = P.run_program(self._main_program, vals)
        d = self.d
        thn = np.ones(d + 3)
        thn[:d] = np.asarray(nkp["k_noise_length"], dtype=np.float64).reshape(-1)[0]     # one noise lengthscale
        thn[d], thn[d + 1] = float(np.asarray(nkp["k_noise_scale"]).reshape(-1)[0]), 0.0
        th = np.ones(d + 3)
        ell = np.asarray(kp["k_length"], dtype=np.float64).reshape(-1)
        th[:d] = np.broadcast_to(ell, (d,)) if ell.size in (1, d) else np.nan
        th[d], th[d + 1] = float(np.asarray(kp["k_scale"]).reshape(-1)[0]), 0.0
        if self.kind == "Periodic":
            if kp.get("period") is None:
                raise ValueError("the Periodic kernel needs 'period' in the dict kernel_prior returns")
            th[d + 2] = float(np.asarray(kp["period"]).reshape(-1)[0])
        mean = np.asarray(self.m.mean_fn(self.X, mp), dtype=np.float64).squeeze() if self.mean_params else self.fixed_mean
        mu_n = self.fixed_mu_n
        if self.noise_mean_params:
            with np.errstate(divide="ignore", invalid="ignore"):
                mu_n = np.log(np.asarray(self.m.noise_mean_fn(self.X, nmp), dtype=np.float64)).squeeze()
        return th, thn, mean, mu_n, {**s1, **s2}

    def _valid(self, th, thn, mean, mu_n):
        ok = np.all(np.isfinite(th)) and np.all(th[:self.d + 1] > 0) and np.all(np.isfinite(thn)) and np.all(thn[:self.d + 1] > 0)
        ok = ok and (self.kind != "Periodic" or th[self.d + 2] > 0)
        return bool(ok and (mean is None or np.all(np.isfinite(mean))) and (mu_n is None or np.all(np.isfinite(mu_n))))

    def _log_prior(self, u, sites, jacobian, want_grad=True):
        val, grad = 0.0, np.zeros(self.dim)
        for s0, sl in self.blocks:
            pr, uu = sites[s0.name].prior, u[sl]
            t = np.asarray(pr.transform(uu), dtype=np.float64)
            val += float(np.sum(pr.log_prob(t)))
            if want_grad:
                grad[sl] = np.asarray(pr.dlog_prob(t)) * np.asarray(pr.dtheta_du(uu))
            if jacobian:
                val += float(np.sum(pr.log_abs_jac(uu)))
                if want_grad:
                    grad[sl] += np.asarray(pr.dlog_abs_jac(uu))
        return val, grad

    # ---- the log joint
    def init_u(self):
        """init_to_median on the program sites; log_var at the default route's start, log(0.1 var(y)).  When the programs
        give an invalid point at the medians (a noise mean a + b x is 0 at a = b = 0), up to INIT_TRIES points uniform in
        (-2, 2) on the unconstrained scale of the program sites (NumPyro's init_to_uniform fallback), from a fixed seed so
        that every chain and chain method starts alike.  Host programs only: no likelihood is evaluated."""
        if self._u0 is None:
            u = np.zeros(self.dim)
            for s, sl in self.blocks:
                u[sl] = float(s.prior.inverse(s.prior.median()))
            u[self.lv] = np.log(0.1 * np.var(self.y0) + 1e-8)
            rng = np.random.default_rng(0)
            for _ in range(self.INIT_TRIES):
                if self._valid(*self._run(u)[:4]):
                    break
                u[self.prog_idx] = rng.uniform(-2.0, 2.0, len(self.prog_idx))
            self._u0 = u
        return self._u0.copy()

    def __call__(self, u, jacobian):
        u = np.asarray(u, dtype=np.float64)
        run = self._run(u)
        self.n_evals += 1
        if not self._valid(*run[:4]):
            return -np.inf, np.zeros(self.dim)
        th, thn, mean, mu_n, _ = run
        lv = u[self.lv]
        ctx = self.m.ctx
        vA, gA, alphaA, infoA = ctx.mll(self.nkind, self.X, lv if mu_n is None else lv - mu_n, thn, self.jitter, True, True)
        vB, gB, alphaB, infoB, gnv = ctx.mll(self.kind, self.X, self.y0 if mean is None else self.y0 - mean, th, self.jitter, True,
                                             self.mean_params, np.exp(lv))
        return self._joint(u, run, vA, gA, alphaA, infoA, vB, gB, alphaB, infoB, gnv, jacobian)

    def batch(self, U, jacobian):
        """the rows of U (one per chain of a vectorized NUTS round): the host programs per row, then one b2gp_mll_draws
        call (noise GP) and one b2gp_mll_draws_v call (main GP) over the valid rows; row r is self(U[r], jacobian) bit for
        bit"""
        U = np.asarray(U, dtype=np.float64)
        runs = [self._run(u) for u in U]
        self.n_evals += len(U)
        out = [(-np.inf, np.zeros(self.dim))] * len(U)
        live = [r for r, run in enumerate(runs) if self._valid(*run[:4])]
        if live:
            ctx = self.m.ctx
            LV = [U[r][self.lv] for r in live]
            RA = np.stack([lv if runs[r][3] is None else lv - runs[r][3] for r, lv in zip(live, LV)])
            RB = np.stack([self.y0 if runs[r][2] is None else self.y0 - runs[r][2] for r in live])
            vA, GA, AA, iA = ctx.mll_draws(self.nkind, self.X, RA, np.stack([runs[r][1] for r in live]), self.jitter,
                                           want_grad=True, want_alpha=True)
            vB, GB, AB, GNV, iB = ctx.mll_draws_v(self.kind, self.X, RB, np.stack([runs[r][0] for r in live]),
                                                  np.stack([np.exp(lv) for lv in LV]), self.jitter, want_grad=True,
                                                  want_alpha=self.mean_params)
            for j, r in enumerate(live):
                out[r] = self._joint(U[r], runs[r], float(vA[j]), GA[j], AA[j], int(iA[j]), float(vB[j]), GB[j],
                                     None if AB is None else AB[j], int(iB[j]), GNV[j], jacobian)
        return np.array([o[0] for o in out]), np.stack([o[1] for o in out])

    @staticmethod
    def _dval_dth(th, g):
        """d value / d theta from d value / d log(theta); the noise slot (0) is a constant"""
        out = np.zeros_like(th)
        nz = th != 0
        out[nz] = g[nz] / th[nz]
        return out

    def _joint(self, u, run, vA, gA, alphaA, infoA, vB, gB, alphaB, infoB, gnv, jacobian):
        if infoA != 0 or infoB != 0 or not (np.isfinite(vA) and np.isfinite(vB)):
            return -np.inf, np.zeros(self.dim)
        th, thn, mean, mu_n, sites = run
        # site densities: analytic gradient, unless the programs are hierarchical (then differenced below)
        lp, grad = self._log_prior(u, sites, jacobian, want_grad=not self.hierarchical)
        grad[self.lv] = -alphaA + gnv * np.exp(u[self.lv])
        dB, dA = self._dval_dth(th, gB), self._dval_dth(thn, gA)
        h = self.FD_STEP
        for k in self.prog_idx:
            e = np.zeros(self.dim)
            e[k] = h
            thp, thnp, mp_, mup, sp = self._run(u + e)
            thm, thnm, mm_, mum, sm_ = self._run(u - e)
            grad[k] += float(np.dot(dB, (thp - thm) / (2 * h))) + float(np.dot(dA, (thnp - thnm) / (2 * h)))
            if self.mean_params:
                grad[k] += float(np.dot(alphaB, (mp_ - mm_) / (2 * h)))
            if self.noise_mean_params:
                grad[k] += float(np.dot(alphaA, (mup - mum) / (2 * h)))
            if self.hierarchical:
                grad[k] += (self._log_prior(u + e, sp, jacobian, False)[0] - self._log_prior(u - e, sm_, jacobian, False)[0]) / (2 * h)
        return vA + vB + lp, grad

    def to_dict(self, U):
        """program sites and log_var in u's order, shaped as sampled; noise 0 (the main kernel's noise, hskgp.py:147)"""
        U = np.atleast_2d(U)
        out = {}
        for s in self.pre:
            out[s.name] = None
        out["log_var"] = U[:, self.lv]
        for s in self.post:
            out[s.name] = None
        for s, sl in self.blocks:
            out[s.name] = np.stack([np.asarray(s.prior.transform(u[sl])).reshape(s.shape) for u in U])
        out["noise"] = np.zeros(len(U))
        return out


# ---------------------------------------------------------------------------------------------- vExactGP
class vExactGP(ExactGP):
    """Gaussian process for vector-valued targets -- gpax/models/vgp.py:23-70: X_train [B, N, d], y_train [B, N], every
    parameter with a leading task axis B; the B posteriors are the members of one batched GPU call."""

    def _set_data(self, X, y=None):
        """vgp.py:199-210."""
        X = np.asarray(X)
        X = X[..., None] if X.ndim == 2 else X
        if y is not None:
            y = np.asarray(y)
            if y.shape[0] != X.shape[0]:
                raise AssertionError("Task dimensions must be identical in inputs and targets")
            return X, y
        return X

    def _members(self, X_new, params, S, noiseless, want, eps=None, **kwargs):
        """S hyper-parameter draws x B tasks = S*B members of one b2gp_posterior_batch call.  params[k] is [S, B, ...]."""
        _need_fused(self)
        X = np.asarray(self.X_train, dtype=np.float64)
        y = np.asarray(self.y_train, dtype=np.float64)
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        B, N, d = X.shape
        Pn = Xn.shape[1]
        flat = {k: np.asarray(v, dtype=np.float64).reshape((S * B,) + np.asarray(v).shape[2:]) for k, v in params.items()
                if v is not None and k in ("k_length", "k_scale", "noise", "period")}
        theta = _theta_rows(flat, d, True)
        yres, pm = y, None
        if self.mean_fn is not None:                                                          # vgp.py:157-166
            get = (lambda x, s: self.mean_fn(x, {k: np.asarray(v)[s] for k, v in params.items()})) if self.mean_fn_prior \
                else (lambda x, s: self.mean_fn(x))
            mX = np.stack([np.asarray(get(X, s)).squeeze() for s in range(S)]).reshape(S, B, N)
            pm = np.stack([np.asarray(get(Xn, s)).squeeze() for s in range(S)]).reshape(S, B, Pn)
            yres = (y[None] - mX).reshape(S * B, N)
        else:
            yres = np.broadcast_to(y[None], (S, B, N)).reshape(S * B, N)
        Xm = np.broadcast_to(X[None], (S, B, N, d)).reshape(S * B, N, d)
        Xnm = np.broadcast_to(Xn[None], (S, B, Pn, d)).reshape(S * B, Pn, d)
        out = self.ctx.posterior(self._fused, Xm, yres, Xnm, theta, noiseless, float(kwargs.get("jitter", 1e-6)), want, eps)
        for k in ("mean", "var", "cov", "y_sampled"):
            if out[k] is not None:
                out[k] = out[k].reshape((S, B) + out[k].shape[1:])
        if pm is not None and out["mean"] is not None:
            out["mean"] = out["mean"] + pm
            if out["y_sampled"] is not None:
                out["y_sampled"] = out["y_sampled"] + pm[:, :, None, :]
        return out

    def fit(self, rng_key, X, y, num_warmup: int = 2000, num_samples: int = 2000, num_chains: int = 1,
            chain_method: str = "sequential", progress_bar: bool = True, print_summary: bool = True, device=None,
            rng_key_predict=None, **kwargs: float) -> None:
        """vgp.py:55-121 under NUTS: one GP per task, every site with a task axis; each log-joint evaluation is one
        b2gp_mll_batch call over the B tasks."""
        from .inference import run_nuts
        X, y = self._set_data(X, y)
        self.X_train, self.y_train = X, y
        lj = _VExactLogJoint(self, kwargs.get("jitter", 1e-6))
        self.mcmc = run_nuts(lj, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method)
        if print_summary:
            self._print_summary()

    def predict_in_batches(self, rng_key, X_new, batch_size: int = 100, samples=None, n: int = 1,
                           filter_nans: bool = False, predict_fn=None, noiseless: bool = False, device=None,
                           **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """vgp.py:175-196: X_new [B, P, d] split along the point axis; means [B, P] and samples [S, n, B, P] joined on it."""
        X_new = self._set_data(X_new)
        y_pred, y_sampled = self._predict_in_batches(rng_key, X_new, batch_size, 1, samples, n, filter_nans, predict_fn,
                                                     noiseless, device, **kwargs)
        return np.concatenate(y_pred, -1), np.concatenate(y_sampled, -1)

    def get_mvn_posterior(self, X_new, params: Dict[str, np.ndarray], noiseless: bool = False,
                          **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """vgp.py:147-172: (mean [B, P], cov [B, P, P]) for a single sample of the parameters (each with a task axis)."""
        one = {k: (None if v is None else np.asarray(v)[None]) for k, v in params.items()}
        out = self._members(X_new, one, 1, noiseless, ("mean", "cov"), **kwargs)
        return out["mean"][0], out["cov"][0]

    def predict(self, rng_key, X_new, samples: Optional[Dict[str, np.ndarray]] = None, n: int = 1, filter_nans: bool = False,
                noiseless: bool = False, device=None, **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """ExactGP.predict over the task-batched posterior: (mean over draws [B, P], y_sampled [S, n, B, P])."""
        X_new = self._set_data(X_new)
        if samples is None:
            samples = self.get_samples(chain_dim=False)
        S = len(next(iter(samples.values())))
        B, Pn = X_new.shape[0], X_new.shape[1]
        eps = posterior_eps(rng_key, S, n * B, Pn, _eps_dtype()).reshape(S, n, B, Pn).transpose(0, 2, 1, 3).reshape(S * B, n, Pn)
        out = self._members(X_new, samples, S, noiseless, ("mean",), eps=eps, **kwargs)
        y_sampled = out["y_sampled"].transpose(0, 2, 1, 3)                                    # [S, n, B, P]
        if filter_nans:
            y_sampled = y_sampled[[i for i in range(S) if not np.isnan(y_sampled[i]).any()]]
        return out["mean"].mean(0), y_sampled


class _VExactLogJoint:
    """log joint of vExactGP.model (vgp.py:55-121) over u = [log k_length (B*d), u k_scale (B), u noise (B)[, log period
    (B)]].  The B per-task likelihoods and their gradients are one b2gp_mll_batch call.  The priors are wired as
    vgp.py:101-121 writes them: k_length is always LogNormal(0, 1), `lengthscale_prior_dist` is the prior of k_scale, and
    `noise_prior_dist` that of noise (vgp.py:92-99)."""

    def __init__(self, model, jitter):
        if model._fused is None:
            raise NotImplementedError("vExactGP.fit: callable kernels are not supported; use 'RBF', 'Matern' or 'Periodic'")
        if model.kernel_prior is not None or model.noise_prior is not None:
            raise NotImplementedError("vExactGP.fit: kernel_prior / noise_prior programs are not interpreted")
        if model.mean_fn_prior is not None:
            raise NotImplementedError("vExactGP.fit: mean_fn_prior (a probabilistic mean function) is not supported")
        self.m, self.jitter, self.kind = model, float(jitter), model._fused
        X = np.asarray(model.X_train, dtype=np.float64)
        self.X = X if X.ndim == 3 else X[..., None]
        self.B, self.N, self.d = self.X.shape
        y = np.asarray(model.y_train, dtype=np.float64).reshape(self.B, self.N)
        if model.mean_fn is not None:
            y = y - np.asarray(model.mean_fn(self.X), dtype=np.float64).squeeze().reshape(self.B, self.N)
        self.y = y
        B, d = self.B, self.d
        # (site, prior, number of coordinates, theta column(s))
        self.sites = [("k_length", P.LogNormal(0.0, 1.0), B * d, slice(0, d)),
                      ("k_scale", model.lengthscale_prior_dist or P.LogNormal(0.0, 1.0), B, d),
                      ("noise", model.noise_prior_dist or P.LogNormal(0.0, 1.0), B, d + 1)]
        if self.kind == "Periodic":
            self.sites.append(("period", P.LogNormal(0.0, 1.0), B, d + 2))
        for _, pr, _, _ in self.sites:
            if not isinstance(pr, P.Prior):
                raise TypeError("priors must be gpax_b200.priors objects (numpyro distributions cannot be used here)")
        self.off = np.cumsum([0] + [n for _, _, n, _ in self.sites])
        self.dim = int(self.off[-1])
        self.n_evals = 0

    def _blocks(self, u):
        for (name, pr, n, col), a in zip(self.sites, self.off[:-1]):
            yield name, pr, col, slice(int(a), int(a) + n)

    def theta_of(self, u):
        th = np.ones((self.B, self.d + 3))
        for _, pr, col, sl in self._blocks(u):
            th[:, col] = np.asarray(pr.transform(u[sl]), dtype=np.float64).reshape(th[:, col].shape)
        return th

    def init_u(self):
        return np.concatenate([np.full(n, float(pr.inverse(pr.median()))) for _, pr, n, _ in self.sites])

    def __call__(self, u, jacobian):
        th = self.theta_of(u)
        val, g, _, _, info = self.m.ctx.mll_batch(self.kind, self.X, self.y, th, self.jitter, True)
        self.n_evals += 1
        return self._joint(u, th, val, g, info, jacobian)

    def batch(self, U, jacobian):
        """the rows of U (one per chain of a vectorized NUTS round) in one b2gp_mll_batch call over k * B members; each
        member is its own CTA or its own b2gp_mll route, so row r is self(U[r], jacobian) bit for bit"""
        k, B = len(U), self.B
        TH = np.stack([self.theta_of(u) for u in U])
        val, g, _, _, info = self.m.ctx.mll_batch(self.kind, np.tile(self.X, (k, 1, 1)), np.tile(self.y, (k, 1)),
                                                  TH.reshape(k * B, -1), self.jitter, True)
        self.n_evals += k
        out = [self._joint(u, th, val[r * B:(r + 1) * B], g[r * B:(r + 1) * B], info[r * B:(r + 1) * B], jacobian)
               for r, (u, th) in enumerate(zip(U, TH))]
        return np.array([o[0] for o in out]), np.stack([o[1] for o in out])

    def _joint(self, u, th, val, g, info, jacobian):
        """the log joint and its gradient w.r.t. u from the B members' likelihoods at theta(u)"""
        val = float(val.sum())
        if (info != 0).any() or not np.isfinite(val):
            return -np.inf, np.zeros(self.dim)
        grad = np.zeros(self.dim)
        for _, pr, col, sl in self._blocks(u):
            uk = u[sl]
            t, gk = th[:, col].reshape(-1), g[:, col].reshape(-1)            # g is d/dlog(theta)
            dt = np.asarray(pr.dtheta_du(uk), dtype=np.float64)
            val += float(np.sum(pr.log_prob(t)))
            grad[sl] = gk / t * dt + np.asarray(pr.dlog_prob(t)) * dt
            if jacobian:
                val += float(np.sum(pr.log_abs_jac(uk)))
                grad[sl] += pr.dlog_abs_jac(uk)
        return val, grad

    def to_dict(self, U):
        """k_length [S, B, d], k_scale / noise (/ period) [S, B]: the reference's sample shapes"""
        U = np.atleast_2d(U)
        th = np.stack([self.theta_of(u) for u in U])
        d = self.d
        out = {"k_length": th[:, :, :d], "k_scale": th[:, :, d], "noise": th[:, :, d + 1]}
        if self.kind == "Periodic":
            out["period"] = th[:, :, d + 2]
        return out


# ---------------------------------------------------------------------------------------------- UIGP
class UIGP(ExactGP):
    """GP with uncertain inputs -- gpax/models/uigp.py:20-77.  The predict path: every posterior draw carries its own
    training inputs params["X_prime"] (uigp.py:138)."""

    def __init__(self, input_dim: int, kernel, mean_fn: Optional[Callable] = None, kernel_prior: Optional[Callable] = None,
                 mean_fn_prior: Optional[Callable] = None, noise_prior_dist=None, lengthscale_prior_dist=None,
                 sigma_x_prior_dist=None, ctx=None) -> None:
        super().__init__(input_dim, kernel, mean_fn, kernel_prior, mean_fn_prior, None, noise_prior_dist,
                         lengthscale_prior_dist, ctx=ctx)
        self.sigma_x_prior_dist = sigma_x_prior_dist

    def _set_data(self, X, y=None):
        """uigp.py:176-190."""
        X = np.asarray(X)
        X = X if X.ndim > 1 else X[:, None]
        if y is not None:
            if not (X.max() == 1 and X.min() == 0) and not self.sigma_x_prior_dist:
                warnings.warn("The default `sigma_x` prior for uncertain (stochastic) inputs assumes data is normalized to "
                              "(0, 1), which is not the case for your data.", UserWarning)
            return X, np.asarray(y).squeeze()
        return X

    def _uigp_batched(self, X_new, params, batched, noiseless, want, eps=None, **kwargs):
        _need_fused(self)
        y = np.asarray(self.y_train, dtype=np.float64).reshape(-1)
        Xp = np.asarray(params["X_prime"], dtype=np.float64)
        Xp = Xp if batched else Xp[None]
        S, N, d = Xp.shape
        Xn = np.asarray(X_new, dtype=np.float64)
        theta = _theta_rows({k: v for k, v in params.items() if k in ("k_length", "k_scale", "noise", "period")}, d, batched)
        yres = y
        if self.mean_fn is not None:                                                          # uigp.py:141-143
            one = (lambda s: {k: np.asarray(v)[s] for k, v in params.items()}) if batched else (lambda s: params)
            f = (lambda x, s: self.mean_fn(x, one(s))) if self.mean_fn_prior else (lambda x, s: self.mean_fn(x))
            yres = np.stack([y - np.asarray(f(Xp[s], s)).squeeze() for s in range(S)])
        out = self.ctx.posterior(self._fused, Xp, yres, Xn, theta, noiseless, float(kwargs.get("jitter", 1e-6)), want, eps)
        if self.mean_fn is not None and out["mean"] is not None:
            pm = np.stack([np.asarray(f(Xn if Xn.ndim == 2 else Xn[s], s)).squeeze() for s in range(S)])
            out["mean"] = out["mean"] + pm
            if out["y_sampled"] is not None:
                out["y_sampled"] = out["y_sampled"] + pm[:, None, :]
        return out

    def get_mvn_posterior(self, X_new, params: Dict[str, np.ndarray], noiseless: bool = False,
                          **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """uigp.py:131-157."""
        out = self._uigp_batched(self._set_data(X_new), params, False, noiseless, ("mean", "cov"), **kwargs)
        return out["mean"][0], out["cov"][0]

    def fit(self, rng_key, X, y, num_warmup: int = 2000, num_samples: int = 2000, num_chains: int = 1,
            chain_method: str = "sequential", progress_bar: bool = True, print_summary: bool = True, device=None,
            rng_key_predict=None, **kwargs: float) -> None:
        """uigp.py:78-129 under NUTS: sigma_x, the latent inputs X_prime and the kernel parameters; the likelihood and its
        gradient w.r.t. X_prime are one b2gp_mll_batch call per evaluation."""
        from .inference import run_nuts
        X, y = self._set_data(X, y)
        self.X_train, self.y_train = X, y
        lj = _UIGPLogJoint(self, kwargs.get("jitter", 1e-6))
        self.mcmc = run_nuts(lj, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method)
        if print_summary:
            self._print_summary()

    def _print_summary(self):
        """uigp.py:192-194: every site but X_prime"""
        for k, v in self.get_samples(1).items():
            if "X_prime" not in k:
                print(f"{k:>12s}  mean {np.mean(v, axis=(0, 1))}  std {np.std(v, axis=(0, 1))}")

    def predict(self, rng_key, X_new, samples: Optional[Dict[str, np.ndarray]] = None, n: int = 1, filter_nans: bool = False,
                noiseless: bool = False, device=None, **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """gp.py:351-399 over uigp.py:159-174: per draw the test inputs are jittered by the learned sigma_x and averaged
        over the n jitters (X_new_prime = Normal(X_new, sigma_x).sample(n).mean(0)), then the usual posterior + sampling."""
        X_new = np.asarray(self._set_data(X_new), dtype=np.float64)
        if samples is None:
            samples = self.get_samples(chain_dim=False)
        S = len(next(iter(samples.values())))
        Pn, d = X_new.shape
        keys = prng.split(prng.as_key(rng_key), S)
        sig = np.asarray(samples["sigma_x"], dtype=np.float64).reshape(S, -1)
        Xnp = np.stack([X_new + sig[s][None, :] * prng.normal(keys[s], (n, Pn, d), _eps_dtype()).astype(np.float64).mean(0)
                        for s in range(S)])
        eps = posterior_eps(rng_key, S, n, Pn, _eps_dtype())
        out = self._uigp_batched(Xnp, samples, True, noiseless, ("mean",), eps=eps, **kwargs)
        y_sampled = out["y_sampled"]
        if filter_nans:
            y_sampled = y_sampled[[i for i in range(S) if not np.isnan(y_sampled[i]).any()]]
        return out["mean"].mean(0), y_sampled


class _UIGPLogJoint:
    """log joint of UIGP.model (uigp.py:78-129) over u = [u sigma_x (d), X_prime (N*d), u k_length (d), u k_scale, u noise
    [, u period]].  X_prime is real-valued and centred: X_prime ~ Normal(X, sigma_x) per feature, sampled as NumPyro does.
    The likelihood log N(y; 0, K(X_prime) + (noise + jitter) I) with its gradients w.r.t. log theta and X_prime is one
    b2gp_mll_batch call with B = 1; the Normal term's gradients w.r.t. X_prime and sigma_x are closed-form."""

    def __init__(self, model, jitter):
        if model._fused is None:
            raise NotImplementedError("UIGP.fit: callable kernels are not supported; use 'RBF', 'Matern' or 'Periodic'")
        if model.kernel_prior is not None or model.noise_prior is not None:
            raise NotImplementedError("UIGP.fit: kernel_prior / noise_prior programs are not interpreted")
        if model.mean_fn is not None or model.mean_fn_prior is not None:
            raise NotImplementedError("UIGP.fit: mean functions are not supported (their derivative w.r.t. X_prime is not "
                                      "available)")
        self.m, self.jitter, self.kind = model, float(jitter), model._fused
        self.X, self.y = model._train_arrays()
        self.N, self.d = self.X.shape
        d = self.d
        self.sx_prior = model.sigma_x_prior_dist or P.HalfNormal(0.1)                     # uigp.py:113-116
        kp = [model.lengthscale_prior_dist or P.LogNormal(0.0, 1.0)] * d + [P.LogNormal(0.0, 1.0)]   # gp.py:235-244
        kidx = list(range(d + 1))
        if self.kind == "Periodic":
            kp.append(P.LogNormal(0.0, 1.0))
            kidx.append(d + 2)
        kp.append(model.noise_prior_dist or P.LogNormal(0.0, 1.0))                         # gp.py:222-227
        kidx.append(d + 1)
        self.kpriors, self.kidx = kp, kidx
        for pr in [self.sx_prior] + kp:
            if not isinstance(pr, P.Prior):
                raise TypeError("priors must be gpax_b200.priors objects (numpyro distributions cannot be used here)")
        self.nx = self.N * d
        self.k0 = d + self.nx                    # first kernel coordinate
        self.dim = self.k0 + len(kp)
        self.n_evals = 0

    def _split(self, u):
        d = self.d
        sx = np.asarray(self.sx_prior.transform(u[:d]), dtype=np.float64)
        Xp = u[d:self.k0].reshape(self.N, d)
        th = np.ones(d + 3)
        for k, (pr, i) in enumerate(zip(self.kpriors, self.kidx)):
            th[i] = pr.transform(u[self.k0 + k])
        return sx, Xp, th

    def init_u(self):
        """init_to_median: X_prime at X, every other site at its prior median"""
        pr = self.sx_prior
        return np.concatenate([np.full(self.d, float(pr.inverse(pr.median()))), self.X.reshape(-1),
                               [float(p.inverse(p.median())) for p in self.kpriors]])

    def __call__(self, u, jacobian):
        sx, Xp, th = self._split(u)
        val, g, _, gx, info = self.m.ctx.mll_batch(self.kind, Xp[None], self.y[None], th[None], self.jitter, True, False, True)
        self.n_evals += 1
        return self._joint(u, sx, Xp, th, val, g, gx, info, jacobian)

    def batch(self, U, jacobian):
        """the rows of U (one per chain of a vectorized NUTS round) as the members of one b2gp_mll_batch call; each member
        is its own CTA or its own b2gp_mll route, so row r is self(U[r], jacobian) bit for bit"""
        parts = [self._split(u) for u in U]
        val, g, _, gx, info = self.m.ctx.mll_batch(self.kind, np.stack([p[1] for p in parts]), np.tile(self.y, (len(U), 1)),
                                                   np.stack([p[2] for p in parts]), self.jitter, True, False, True)
        self.n_evals += len(U)
        out = [self._joint(u, sx, Xp, th, val[r:r + 1], g[r:r + 1], gx[r:r + 1], info[r:r + 1], jacobian)
               for r, (u, (sx, Xp, th)) in enumerate(zip(U, parts))]
        return np.array([o[0] for o in out]), np.stack([o[1] for o in out])

    def _joint(self, u, sx, Xp, th, val, g, gx, info, jacobian):
        """the log joint and its gradients from the likelihood at (X_prime, theta) (b2gp_mll_batch's outputs, one member)"""
        d = self.d
        val = float(val[0])
        if info[0] != 0 or not np.isfinite(val) or not np.all(np.isfinite(sx)) or not np.all(sx > 0):
            return -np.inf, np.zeros(self.dim)
        grad = np.zeros(self.dim)
        # X_prime ~ Normal(X, sigma_x): value, d/dX_prime, d/dsigma_x
        r = (Xp - self.X) / sx
        val += float(np.sum(-0.5 * r * r - np.log(sx) - 0.5 * math.log(2 * math.pi)))
        grad[d:self.k0] = (gx[0] - r / sx).reshape(-1)
        dsx = np.sum(r * r, axis=0) / sx - self.N / sx
        pr, us = self.sx_prior, u[:d]
        dt = np.asarray(pr.dtheta_du(us), dtype=np.float64)
        val += float(np.sum(pr.log_prob(sx)))
        grad[:d] = dsx * dt + np.asarray(pr.dlog_prob(sx)) * dt
        if jacobian:
            val += float(np.sum(pr.log_abs_jac(us)))
            grad[:d] += pr.dlog_abs_jac(us)
        for k, (pr, i) in enumerate(zip(self.kpriors, self.kidx)):
            uk, t = u[self.k0 + k], th[i]
            dt = float(pr.dtheta_du(uk))
            val += float(pr.log_prob(t))
            grad[self.k0 + k] = g[0, i] / t * dt + float(pr.dlog_prob(t)) * dt       # g is d/dlog(theta)
            if jacobian:
                val += float(pr.log_abs_jac(uk))
                grad[self.k0 + k] += float(pr.dlog_abs_jac(uk))
        return val, grad

    def to_dict(self, U):
        """sigma_x [S, d], X_prime [S, N, d], k_length [S, d], k_scale / noise (/ period) [S]"""
        U = np.atleast_2d(U)
        parts = [self._split(u) for u in U]
        th = np.stack([p[2] for p in parts])
        d = self.d
        out = {"sigma_x": np.stack([p[0] for p in parts]), "X_prime": np.stack([p[1] for p in parts]),
               "k_length": th[:, :d], "k_scale": th[:, d], "noise": th[:, d + 1]}
        if self.kind == "Periodic":
            out["period"] = th[:, d + 2]
        return out
