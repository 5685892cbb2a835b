"""
dkl.py -- deep kernel learning with the reference's surface: `viDKL` (gpax/models/vidkl.py:71-397) and the fully Bayesian
`DKL` (gpax/models/dkl.py:69-150).  The GP runs on the embedding z = MLP(X).  Every numerical step is on the GPU:
b2gp_mlp_forward embeds inputs for any number of weight sets, b2gp_dkl_mll evaluates the likelihood log N(y; 0, K(z)) and
its gradient w.r.t. the kernel hyper-parameters and, through the network's backward pass, every weight and bias, and
b2gp_posterior predicts on the embeddings; b2gp_dkl_posterior_grad gives the posterior's gradient w.r.t. the raw test
inputs, which acquisition.optimize_acq uses for single-channel viDKL and DKL.  The optimiser (viDKL: Adam with b1 = 0.5,
inference.adam) and the sampler (DKL: NUTS, inference.run_nuts) are the host-side loops the other models use.

The feature extractor is the reference's default MLP only: viDKL's ReLU MLP 64 -> 64 -> z_dim (vidkl.py:400-412) and DKL's
tanh MLP over `hidden_dim` (dkl.py:167-177).  Custom haiku modules or callables, `latent_prior` and custom `nn_prior`
programs are refused, and so are `kernel_prior` programs (priors on the kernel sites go through `lengthscale_prior_dist` /
`noise_prior_dist`): a program would have to be re-run and differenced on the host per step, as ExactGP's ProgramLogJoint
does, and that path is not wired to b2gp_dkl_mll.

Initialisation (seeded from `rng_key`; bitwise equality with a JAX run is not a goal):
  * kernel sites: the exact median of their prior, as fit_vi_gp does for viGP;
  * network sites with nn_prior=True: AutoDelta's init_to_median, i.e. per element the median of 15 draws from the prior
    (the exact median, 0, would start every weight at 0 and leave the network without a gradient);
  * nn_prior=False: haiku's default, TruncatedNormal(stddev = 1 / sqrt(fan_in)) cut at two standard deviations, zero bias.
"""
import math
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import _ffi
from . import priors as P
from . import prng
from .gp import ExactGP, _eps_dtype, _theta_rows
from .utils import posterior_eps, seed_from_key

INIT_MEDIAN_DRAWS = 15        # numpyro's init_to_median(num_samples=15), AutoDelta's default init strategy


def _refuse(nn, latent_prior, input_dim, nn_prior_program=None):
    if nn is not None:
        raise NotImplementedError("custom feature extractors (haiku modules, callables) are not supported: the MLP is built in")
    if latent_prior is not None:
        raise NotImplementedError("latent_prior is not supported")
    if nn_prior_program is not None:
        raise NotImplementedError("custom nn_prior programs are not supported: Normal(0, 1) weights and Cauchy(0, 1) biases")
    if isinstance(input_dim, (tuple, list)):
        if len(input_dim) != 1:
            raise NotImplementedError("input_dim must be an int or (D,): the MLP takes flat feature vectors")
        return int(input_dim[0])
    return int(input_dim)


def _nn_log_prior(wmask, flat):
    """log p of the network sites with Normal(0, 1) weights and Cauchy(0, 1) biases (vidkl.py:93-96) and its gradient"""
    normal, cauchy = P.Normal(0.0, 1.0), P.Cauchy(0.0, 1.0)
    val = float(np.sum(normal.log_prob(flat[wmask]))) + float(np.sum(cauchy.log_prob(flat[~wmask])))
    return val, np.where(wmask, normal.dlog_prob(flat), cauchy.dlog_prob(flat))


class _MLPModel(ExactGP):
    """What viDKL and DKL share: the layer widths, the kernel sites and the embedding on the GPU."""

    act = _ffi.ACT_RELU

    def _setup(self, D, widths, kwargs):
        self.data_dim = (D,)
        self.widths = [int(w) for w in widths]
        self.kernel_dim = self.widths[-1]
        if self._fused is None:
            raise NotImplementedError("deep kernel learning needs kernel 'RBF', 'Matern' or 'Periodic'")
        if self.kernel_dim > 16:
            raise ValueError("z_dim must be <= 16")
        self.noise_prior_dist = kwargs.get("noise_prior_dist")
        self.lengthscale_prior_dist = kwargs.get("lengthscale_prior_dist")

    def _shapes(self):
        """[(in, out)] per layer"""
        ins = [self.data_dim[0]] + self.widths[:-1]
        return list(zip(ins, self.widths))

    def _kernel_sites(self):
        """(name, prior, theta index) of the kernel and noise sites (gp.py:222-247)"""
        d = self.kernel_dim
        lp = self.lengthscale_prior_dist or P.LogNormal(0.0, 1.0)
        s = [("k_length", lp, k) for k in range(d)] + [("k_scale", P.LogNormal(0.0, 1.0), d),
                                                       ("noise", self.noise_prior_dist or P.LogNormal(0.0, 1.0), d + 1)]
        if self._fused == "Periodic":
            s.append(("period", P.LogNormal(0.0, 1.0), d + 2))
        return s

    def _theta(self, u):
        th = np.ones(self.kernel_dim + 3)
        for k, (_, pr, i) in enumerate(self._kernel_sites()):
            th[i] = pr.transform(u[k])
        return th

    def _kernel_dict(self, th):
        d = self.kernel_dim
        out = {"k_length": th[..., :d], "k_scale": th[..., d], "noise": th[..., d + 1]}
        if self._fused == "Periodic":
            out["period"] = th[..., d + 2]
        return out

    def _embed(self, X, flat):
        """Z [S, N, d] for flat parameter rows [S, P]"""
        X = np.asarray(self._set_data(X), dtype=np.float64)
        return self.ctx.mlp_forward(X, self.widths, self.act, np.atleast_2d(flat))

    def _posterior(self, X_new, flat, theta, yres, noiseless, want, eps=None, jitter=1e-6):
        """the batched posterior on the embeddings of S weight sets: flat [S, P], theta [S, d+3], yres [N] or [S, N]"""
        Ztr = self._embed(self.X_train, flat)
        Zn = self._embed(X_new, flat)
        return self.ctx.posterior(self._fused, Ztr, yres, Zn, theta, noiseless, jitter, want, eps)

    def _posterior_batched(self, X_new, params, batched, noiseless, want, eps=None, **kwargs):
        """The seam the acquisition functions and ExactGP._predict call (acquisition.kg / KG / qEI / qUCB / qPOI / qKG):
        ExactGP's version would run the GP on the raw inputs, here it is the posterior on the embeddings of one
        (batched=False) or S (batched=True) parameter sets."""
        flat, kp = self._split_params(params)
        th = _theta_rows(kp, self.kernel_dim, batched)
        y = np.asarray(self.y_train, dtype=np.float64)
        return self._posterior(X_new, np.atleast_2d(flat), th, y if y.ndim == 2 else y.reshape(-1), noiseless, want, eps,
                               float(kwargs.get("jitter", 1e-6)))

    def _posterior_grad(self, X_new, params, batched, noiseless, **kwargs):
        """Per-draw posterior mean [S, P], variance [S, P] and their gradients dmean, dvar [S, P, D] w.r.t. the RAW test
        inputs (b2gp_dkl_posterior_grad: the posterior gradient on the embedding pulled back through the network), for
        one (batched=False: viDKL's (nn_params, kernel_params)) or S (batched=True: DKL's draws) parameter sets.  Single-
        channel targets only; acquisition.optimize_acq calls it for viDKL and DKL."""
        y = np.asarray(self.y_train, dtype=np.float64)
        if y.ndim != 1:
            raise NotImplementedError("posterior gradients of a multi-channel model are not supported")
        flat, kp = self._split_params(params)
        th = _theta_rows(kp, self.kernel_dim, batched)
        X = np.asarray(self._set_data(self.X_train), dtype=np.float64)
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        out = self.ctx.dkl_posterior_grad(self._fused, X, y, Xn, self.widths, self.act, np.atleast_2d(flat), th, noiseless,
                                          float(kwargs.get("jitter", 1e-6)))
        return out["mean"], out["var"], out["dmean"], out["dvar"]


# ------------------------------------------------------------------------------------------------------------ viDKL
class viDKL(_MLPModel):
    """
    Variational deep kernel learning (gpax/models/vidkl.py): a 3-layer ReLU MLP (64, 64, z_dim) embeds the inputs, an exact
    GP runs on the embedding; the network weights and the kernel hyper-parameters are fitted jointly by SVI (Adam with
    b1 = 0.5, AutoDelta or AutoNormal guide).  `nn_params` use haiku's layout, {"mlp/~/linear": {"w": [in, out], "b": [out]},
    "mlp/~/linear_1": ..., "mlp/~/linear_2": ...}, so weights trained by the reference predict here unchanged.
    """

    HIDDEN = (64, 64)
    INTERNAL_BATCH = 8192

    def __init__(self, input_dim, z_dim: int = 2, kernel: str = "RBF", kernel_prior=None, nn=None, nn_prior: bool = True,
                 latent_prior=None, guide: str = "delta", ctx=None, **kwargs) -> None:
        D = _refuse(nn, latent_prior, input_dim)
        if kernel_prior is not None:
            raise NotImplementedError("kernel_prior programs are not supported by viDKL; use lengthscale_prior_dist / "
                                      "noise_prior_dist")
        if guide not in ["delta", "normal"]:
            raise NotImplementedError("Select guide between 'delta' and 'normal'")
        super().__init__(D, kernel, ctx=ctx)
        self._setup(D, list(self.HIDDEN) + [int(z_dim)], kwargs)
        self.nn_prior = bool(nn_prior)
        self.guide_type = guide
        self.kernel_params = None
        self.nn_params = None
        self.loss = None

    def _split_params(self, params):
        nn_params, k_params = params
        return self.to_flat(nn_params), k_params

    # ---- haiku layout <-> the flat C-ABI layout (per layer W [in, out] row-major, then b)
    @staticmethod
    def _layer_names(n):
        return ["mlp/~/linear"] + [f"mlp/~/linear_{i}" for i in range(1, n)]

    def to_flat(self, nn_params) -> np.ndarray:
        """haiku dict -> flat parameters; a leading channel axis C on every leaf gives [C, P]"""
        names = self._layer_names(len(self.widths))
        w0 = np.asarray(nn_params[names[0]]["w"])
        lead = w0.shape[:-2]
        parts = []
        for name in names:
            w, b = np.asarray(nn_params[name]["w"], np.float64), np.asarray(nn_params[name]["b"], np.float64)
            parts += [w.reshape(lead + (-1,)), b.reshape(lead + (-1,))]
        return np.concatenate(parts, axis=-1)

    def from_flat(self, flat) -> Dict[str, Dict[str, np.ndarray]]:
        flat = np.asarray(flat, dtype=np.float64)
        lead, out, o = flat.shape[:-1], {}, 0
        for name, (i, w) in zip(self._layer_names(len(self.widths)), self._shapes()):
            W = flat[..., o:o + i * w].reshape(lead + (i, w))
            o += i * w
            out[name] = {"w": W, "b": flat[..., o:o + w]}
            o += w
        return out

    # ---- fit
    def _init_params(self, rng):
        """(u_theta, flat network parameters) at the start of the fit (see the module docstring)"""
        u = np.array([float(pr.inverse(pr.median())) for _, pr, _ in self._kernel_sites()])
        return u, self._init_network(rng)

    def _init_network(self, rng):
        """the flat network parameters at the start of the fit"""
        parts = []
        for i, w in self._shapes():
            if self.nn_prior:
                W = np.median(rng.standard_normal((INIT_MEDIAN_DRAWS, i, w)), axis=0)
                b = np.median(rng.standard_cauchy((INIT_MEDIAN_DRAWS, w)), axis=0)
            else:
                W = rng.standard_normal((i, w))
                while np.any(np.abs(W) > 2.0):
                    bad = np.abs(W) > 2.0
                    W[bad] = rng.standard_normal(int(bad.sum()))
                W, b = W / math.sqrt(i), np.zeros(w)
            parts += [W.ravel(), b]
        return np.concatenate(parts)

    def _weight_mask(self):
        """True at the weights, False at the biases of the flat layout"""
        return np.concatenate([np.r_[np.ones(i * w), np.zeros(w)] for i, w in self._shapes()]).astype(bool)

    def _mlp_inputs(self, X):
        """the network's input rows of a (2-d) input array"""
        return X

    def _log_joint(self, X, Xd, yd, jitter):
        """log p(y, sites) over (u_theta, flat) and its gradient; priors on theta in the constrained space without the
        Jacobian (as fit_vi_gp), Normal(0, 1) weights and Cauchy(0, 1) biases when nn_prior (vidkl.py:93-96).  X: the
        host inputs, Xd / yd: the network's inputs and the targets on the device."""
        sites = self._kernel_sites()
        nth = len(sites)
        wmask = self._weight_mask()

        def f(v, jacobian=False):
            u, flat = v[:nth], v[nth:]
            th = self._theta(u)
            val, g, gp, _, info = self.ctx.dkl_mll(self._fused, Xd, yd, self.widths, self.act, flat, th, jitter)
            if info != 0 or not np.isfinite(val):
                return -np.inf, np.zeros_like(v)
            gu = np.zeros(nth)
            for k, (_, pr, i) in enumerate(sites):
                t, dt = th[i], float(pr.dtheta_du(u[k]))
                val += float(pr.log_prob(t))
                gu[k] = g[i] / t * dt + float(pr.dlog_prob(t)) * dt
                if jacobian:
                    val += float(pr.log_abs_jac(u[k]))
                    gu[k] += float(pr.dlog_abs_jac(u[k]))
            if self.nn_prior:
                lp, glp = _nn_log_prior(wmask, flat)
                val += lp
                gp = gp + glp
            return val, np.concatenate([gu, gp])
        return f, nth

    def single_fit(self, rng_key, X, y, num_steps: int = 1000, step_size: float = 5e-3, print_summary: bool = True,
                   progress_bar=True, **kwargs):
        """vidkl.py:126-161: returns (nn_params, kernel_params, losses) of one fit"""
        from .inference import adam
        X = np.asarray(self._set_data(X), dtype=np.float64)
        y = np.asarray(y, dtype=np.float64).reshape(-1)
        rng = seed_from_key(rng_key)
        Xd, yd = self.ctx.to_device(self._mlp_inputs(X)), self.ctx.to_device(y)       # uploaded once for the whole fit
        try:
            f, nth = self._log_joint(X, Xd, yd, float(kwargs.get("jitter", 1e-6)))
            u0, flat0 = self._init_params(rng)
            loc = np.concatenate([u0, flat0])
            dim = loc.size
            normal = self.guide_type == "normal"
            # AutoNormal covers the sample sites: the kernel sites, and the network's only when it has a prior
            # (nn_prior=False makes the weights numpyro.param, point parameters, vidkl.py:97-99)
            nr = dim if self.nn_prior else nth
            params = np.concatenate([loc, np.full(nr, math.log(0.1))]) if normal else loc

            def objective(p):
                if normal:
                    mu, r = p[:dim], p[dim:]
                    e = rng.standard_normal(nr)
                    v = mu.copy()
                    v[:nr] += np.exp(r) * e
                    val, g = f(v, jacobian=True)
                    elbo = val + r.sum() + 0.5 * nr * (1 + math.log(2 * math.pi))
                    return elbo, np.concatenate([g, g[:nr] * e * np.exp(r) + 1.0])
                return f(p)
            params, losses = adam(params, objective, num_steps, step_size, progress_bar)
        finally:
            Xd.free()
            yd.free()
        loc = params[:dim]
        kp = {k: np.asarray(v) for k, v in self._kernel_dict(self._theta(loc[:nth])).items()}
        return self.from_flat(loc[nth:]), kp, np.array(losses)

    def fit(self, rng_key, X, y, num_steps: int = 1000, step_size: float = 5e-3, print_summary: bool = True,
            progress_bar=True, **kwargs):
        """vidkl.py:163-203.  y [N], or [C, N] for C channels fitted independently from the same key (the reference's
        vmap); then every leaf of nn_params / kernel_params carries a leading C axis."""
        X = self._set_data(X)
        y = np.asarray(y)
        self.X_train, self.y_train = X, y
        if y.ndim == 2:
            fits = [self.single_fit(rng_key, X, yi, num_steps, step_size, False, False, **kwargs) for yi in y]
            self.nn_params = {k: {p: np.stack([f[0][k][p] for f in fits]) for p in ("w", "b")} for k in fits[0][0]}
            self.kernel_params = {k: np.stack([f[1][k] for f in fits]) for k in fits[0][1]}
            self.loss = np.stack([f[2] for f in fits])
        else:
            self.nn_params, self.kernel_params, self.loss = self.single_fit(rng_key, X, y, num_steps, step_size, print_summary,
                                                                            progress_bar, **kwargs)
        if print_summary:
            self._print_summary()

    # ---- predict
    def get_mvn_posterior(self, X_new, nn_params, k_params, noiseless: bool = False, y_residual=None,
                          **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """vidkl.py:206-236: mean [P] and covariance [P, P] for one set of network weights and kernel parameters"""
        y = self.y_train if y_residual is None else y_residual
        th = _theta_rows(k_params, self.kernel_dim, False)
        out = self._posterior(X_new, self.to_flat(nn_params), th, np.asarray(y, np.float64).reshape(-1), noiseless,
                              ("mean", "cov"), jitter=float(kwargs.get("jitter", 1e-6)))
        return out["mean"][0], out["cov"][0]

    def sample_from_posterior(self, rng_key, X_new, n: int = 1000, noiseless: bool = False, **kwargs):
        """vidkl.py:238-251"""
        if np.asarray(self.y_train).ndim > 1:
            raise NotImplementedError("Currently does not support a multi-channel regime")
        mean, K = self.get_mvn_posterior(X_new, self.nn_params, self.kernel_params, noiseless, **kwargs)
        eps = posterior_eps(rng_key, 1, n, mean.shape[0], _eps_dtype(), per_draw_keys=False)
        y, _ = self.ctx.mvn_sample(mean[None], K[None], eps)
        return mean, y[0]

    def get_samples(self):
        """vidkl.py:253-255: (nn_params, kernel_params)"""
        return self.nn_params, self.kernel_params

    def predict(self, rng_key, X_new, params=None, noiseless: bool = False, *args, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """vidkl.py:277-318: (mean, var), [P] or, for C channels, [C, P].  The channels go through one b2gp_mlp_forward
        with S = C weight sets and one batched posterior on the per-channel embeddings."""
        nn_params, k_params = (self.nn_params, self.kernel_params) if params is None else params
        X_new = self._set_data(X_new)
        y = np.asarray(self.y_train, dtype=np.float64)
        multi = y.ndim == 2
        th = _theta_rows(k_params, self.kernel_dim, multi)
        out = self._posterior(X_new, self.to_flat(nn_params), th, y, noiseless, ("mean", "var"),
                              jitter=float(kwargs.get("jitter", 1e-6)))
        if multi:
            return out["mean"], out["var"]
        return out["mean"][0], out["var"][0]

    def predict_in_batches(self, rng_key, X_new, batch_size: int = 100, params=None, noiseless: bool = False,
                           **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """vidkl.py:257-275.  Chunks smaller than INTERNAL_BATCH rows are merged before they go to the device, as in
        viGP.predict_in_batches: a test point's (mean, var) does not depend on the other points of its chunk."""
        batch_size = max(int(batch_size), self.INTERNAL_BATCH)
        X_new = self._set_data(X_new)
        if X_new.shape[0] <= batch_size:
            return self.predict(rng_key, X_new, params, noiseless, **kwargs)
        cat_dim = 1 if np.asarray(self.y_train).ndim == 2 else 0
        mean, var = self._predict_in_batches(rng_key, X_new, batch_size, 0, params,
                                             predict_fn=lambda xi: self.predict(rng_key, xi, params, noiseless, **kwargs))
        return np.concatenate(mean, cat_dim), np.concatenate(var, cat_dim)

    def fit_predict(self, rng_key, X, y, X_new, num_steps: int = 1000, step_size: float = 5e-3, n_models: int = 1,
                    batch_size: int = 100, noiseless: bool = False, ensemble_method: str = "vectorized",
                    print_summary: bool = True, progress_bar=True, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """vidkl.py:320-369.  The ensemble's keys are jax.random.split(rng_key, n_models), as in the reference.  Both
        ensemble methods ('vectorized', 'parallel') fit and predict the members one after another on this model's
        device.  Returns (mean, var) of shape [P] / [C, P], with a leading n_models axis when n_models > 1."""
        if n_models > 1 and ensemble_method not in ["vectorized", "parallel"]:
            raise ValueError("For the ensemble_method, select between 'vectorized and 'parallel'.")
        keys = prng.split(rng_key, n_models)

        def single_fit_predict(key):
            self.fit(key, X, y, num_steps, step_size, print_summary, progress_bar, **kwargs)
            return self.predict_in_batches(key, X_new, batch_size, None, noiseless, **kwargs)

        if n_models > 1:
            res = [single_fit_predict(k) for k in keys]
            return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])
        return single_fit_predict(keys[0])

    def embed(self, X_new) -> np.ndarray:
        """vidkl.py:371-384: z [N, d], or [C, N, d] with C channels"""
        flat = self.to_flat(self.nn_params)
        Z = self._embed(X_new, flat)
        return Z if flat.ndim == 2 else Z[0]

    def _print_summary(self) -> None:
        print("\nInferred GP kernel parameters")
        for k, v in self.kernel_params.items():
            print(k, " " * (15 - len(k)), np.around(np.asarray(v), 4))


# ------------------------------------------------------------------------------------------------------------ DKL
class DKLLogJoint:
    """log p(y, sites) of DKL.model (dkl.py:83-111) over the unconstrained vector u = (log theta sites, w0, b0, ..., wL, bL)
    for run_nuts: the likelihood and its gradient w.r.t. theta and every weight from b2gp_dkl_mll, Normal(0, 1) weights
    and Cauchy(0, 1) biases (dkl.py:152-164), LogNormal kernel sites with their Jacobian."""

    def __init__(self, model, rng, jitter=1e-6):
        self.m, self.jitter, self.rng = model, float(jitter), rng
        X, y = model._train_arrays()
        self.Xd, self.yd = model.ctx.to_device(X), model.ctx.to_device(y)
        self.sites = model._kernel_sites()
        self.nth = len(self.sites)
        self.wmask = np.concatenate([np.r_[np.ones(i * w), np.zeros(w)] for i, w in model._shapes()]).astype(bool)
        self.dim = self.nth + self.wmask.size
        self.n_evals = 0

    def close(self):
        self.Xd.free()
        self.yd.free()

    def init_u(self):
        """kernel sites at their prior median, network sites at the median of INIT_MEDIAN_DRAWS prior draws"""
        u = [float(pr.inverse(pr.median())) for _, pr, _ in self.sites]
        net = np.where(self.wmask, np.median(self.rng.standard_normal((INIT_MEDIAN_DRAWS, self.wmask.size)), axis=0),
                       np.median(self.rng.standard_cauchy((INIT_MEDIAN_DRAWS, self.wmask.size)), axis=0))
        return np.concatenate([u, net])

    def __call__(self, u, jacobian):
        m = self.m
        th = m._theta(u[:self.nth])
        flat = u[self.nth:]
        self.n_evals += 1
        val, g, gp, _, info = m.ctx.dkl_mll(m._fused, self.Xd, self.yd, m.widths, m.act, flat, th, self.jitter)
        if info != 0 or not np.isfinite(val):
            return -np.inf, np.zeros(self.dim)
        gu = np.zeros(self.nth)
        for k, (_, pr, i) in enumerate(self.sites):
            t, dt = th[i], float(pr.dtheta_du(u[k]))
            val += float(pr.log_prob(t))
            gu[k] = g[i] / t * dt + float(pr.dlog_prob(t)) * dt
            if jacobian:
                val += float(pr.log_abs_jac(u[k]))
                gu[k] += float(pr.dlog_abs_jac(u[k]))
        normal, cauchy = P.Normal(0.0, 1.0), P.Cauchy(0.0, 1.0)
        val += float(np.sum(normal.log_prob(flat[self.wmask]))) + float(np.sum(cauchy.log_prob(flat[~self.wmask])))
        gp = gp + np.where(self.wmask, normal.dlog_prob(flat), cauchy.dlog_prob(flat))
        return val, np.concatenate([gu, gp])

    def to_dict(self, U):
        U = np.atleast_2d(U)
        th = np.stack([self.m._theta(u[:self.nth]) for u in U])
        out = self.m.from_flat(U[:, self.nth:])
        out.update(self.m._kernel_dict(th))
        return out


class DKL(_MLPModel):
    """
    Fully Bayesian deep kernel learning (gpax/models/dkl.py): a tanh MLP over `hidden_dim` (default [64, 32]) and a linear
    layer to z_dim embed the inputs; NUTS samples the weights (sites w0, b0, ..., w{L}, b{L}: Normal(0, 1) weights,
    Cauchy(0, 1) biases) jointly with the kernel hyper-parameters.
    """

    act = _ffi.ACT_TANH

    def __init__(self, input_dim, z_dim: int = 2, kernel: str = "RBF", kernel_prior=None, nn=None, nn_prior=None,
                 latent_prior=None, hidden_dim: Optional[List[int]] = None, ctx=None, **kwargs) -> None:
        D = _refuse(nn, latent_prior, input_dim, nn_prior)
        if kernel_prior is not None:
            raise NotImplementedError("kernel_prior programs are not supported by DKL; use lengthscale_prior_dist / "
                                      "noise_prior_dist")
        super().__init__(D, kernel, ctx=ctx)
        hdim = list(hidden_dim) if hidden_dim is not None else [64, 32]
        self._setup(D, hdim + [int(z_dim)], kwargs)

    def _split_params(self, params):
        return self.to_flat(params), params

    def site_names(self):
        L = len(self.widths)
        return [n for i in range(L) for n in (f"w{i}", f"b{i}")]

    def to_flat(self, params) -> np.ndarray:
        """site dict -> flat parameters [S, P] (leading draw axis) or [P]"""
        w0 = np.asarray(params["w0"])
        lead = w0.shape[:-2]
        parts = []
        for i in range(len(self.widths)):
            parts += [np.asarray(params[f"w{i}"], np.float64).reshape(lead + (-1,)),
                      np.asarray(params[f"b{i}"], np.float64).reshape(lead + (-1,))]
        return np.concatenate(parts, axis=-1)

    def from_flat(self, flat) -> Dict[str, np.ndarray]:
        flat = np.asarray(flat, dtype=np.float64)
        lead, out, o = flat.shape[:-1], {}, 0
        for l, (i, w) in enumerate(self._shapes()):
            out[f"w{l}"] = flat[..., o:o + i * w].reshape(lead + (i, w))
            o += i * w
            out[f"b{l}"] = flat[..., o:o + w]
            o += w
        return out

    def fit(self, rng_key, X, y, num_warmup: int = 2000, num_samples: int = 2000, num_chains: int = 1,
            chain_method: str = "sequential", progress_bar: bool = True, print_summary: bool = True, device=None,
            rng_key_predict=None, **kwargs) -> None:
        """gp.py:166-220 with DKL.model: NUTS over the network weights and the kernel hyper-parameters (chains run one
        after another)"""
        from .inference import run_nuts
        X, y = self._set_data(X, y)
        self.X_train, self.y_train = X, y
        lj = DKLLogJoint(self, seed_from_key(rng_key), kwargs.get("jitter", 1e-6))
        try:
            self.mcmc = run_nuts(lj, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method)
        finally:
            lj.close()
        if print_summary:
            self._print_summary()

    def get_mvn_posterior(self, X_new, params: Dict[str, np.ndarray], noiseless: bool = False,
                          **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """dkl.py:113-132: mean [P] and covariance [P, P] for one sample of the sites"""
        th = _theta_rows(params, self.kernel_dim, False)
        y = np.asarray(self.y_train, dtype=np.float64).reshape(-1)
        out = self._posterior(X_new, self.to_flat(params), th, y, noiseless, ("mean", "cov"), jitter=float(kwargs.get("jitter", 1e-6)))
        return out["mean"][0], out["cov"][0]

    def predict(self, rng_key, X_new, samples: Optional[Dict[str, np.ndarray]] = None, n: int = 1,
                filter_nans: bool = False, noiseless: bool = False, device=None, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """gp.py:351-399 on every draw: one b2gp_mlp_forward with S = draws, then the batched posterior with mean and
        samples.  Returns (mean over draws [P], y_sampled [S, n, P])."""
        X_new = self._set_data(X_new)
        if samples is None:
            samples = self.get_samples(chain_dim=False)
        flat = np.atleast_2d(self.to_flat(samples))
        S, Pn = flat.shape[0], X_new.shape[0]
        th = _theta_rows(samples, self.kernel_dim, True)
        eps = posterior_eps(rng_key, S, n, Pn, _eps_dtype())
        y = np.asarray(self.y_train, dtype=np.float64).reshape(-1)
        out = self._posterior(X_new, flat, th, y, noiseless, ("mean",), eps=eps, jitter=float(kwargs.get("jitter", 1e-6)))
        y_sampled = out["y_sampled"]
        if filter_nans:
            y_sampled = y_sampled[[i for i in range(S) if not np.isnan(y_sampled[i]).any()]]
        return out["mean"].mean(0), y_sampled

    def embed(self, X_new) -> np.ndarray:
        """dkl.py:134-143: z [S, N, d] for every draw"""
        return self._embed(X_new, self.to_flat(self.get_samples(chain_dim=False)))

    def _print_summary(self):
        s = self.get_samples(chain_dim=False)
        for k in ("k_scale", "k_length", "noise", "period"):
            if k in s:
                v = np.asarray(s[k])
                print(f"{k:>12s}  mean {np.mean(v, axis=0)}  std {np.std(v, axis=0)}")


# ------------------------------------------------------------------------------------------------------------ viMTDKL
class viMTDKL(viDKL):
    """
    Multi-task deep kernel learning (gpax/models/vi_mtdkl.py): viDKL's ReLU MLP (64, 64, z_dim) embeds the inputs and the
    GP on the embedding has the LCM covariance of MultiTaskGP, sum_q (k_q(z, z') + jitter [same point]) B_q[t, t'] with
    B_q = W_q W_q^T + diag(v_q).  The network and the kernel sites are fitted jointly by SVI as in viDKL; the likelihood
    and its gradient w.r.t. every site and weight come from b2gp_mtdkl_mll, the posterior from b2gp_posterior_multitask
    on the embeddings.  Both forms of the reference:
      * multitask form (shared_input_space=False): one row per observation, its task id in the last column of X; the
        network sees X[:, :-1];
      * Kronecker form (shared_input_space=True, needs num_tasks): every task observed at every input, y of length N*T
        in point-major order (point i, task t at i*T + t); predictions have length P*T in the same order.

    Sites (vi_mtdkl.py:163-209): k_length LogNormal(0, 1) [L, z_dim], k_scale Normal(1, 1e-4) [L, 1], W Normal(0, 10)
    [L, T, rank] (or W_prior_dist), v LogNormal(0, 1) [L, T] (or v_prior_dist), noise LogNormal(0, 1) [T] (or
    noise_prior_dist).  `kernel_params` carries them in these shapes.  T defaults to the distinct labels of the task
    column, rank to T - 1.  The kernel sites start at their prior median, except W, whose median 0 is a stationary point
    of the loss (d/dW = (G + G^T) W = 0 there and the prior's gradient is 0 too): W starts, as the network's weights do,
    at the element-wise median of INIT_MEDIAN_DRAWS prior draws (numpyro's init_to_median).

    Differences from the reference: `embed` strips the task column of the multitask form before the network (the
    reference would feed it to the network, whose input width it does not match).  Refused: data_kernel 'Periodic' (the
    reference samples no period, so its own model fails there), data_kernel_prior / task_kernel_prior programs and custom
    networks (as viDKL).  Limits of the GPU path: T <= 8, L <= 4, z_dim <= 16.

    Acquisition functions: EI / UCB / POI / UE work through `predict`; KG works in the multitask form, with the
    candidate's task setting its noise in the rank-1 update (`_kg_terms`), and raises NotImplementedError in the
    Kronecker form; the q-batch functions (qEI, qUCB, qPOI, qKG) need a fully Bayesian model and raise ValueError, as for
    viDKL and in the reference; `acquisition.optimize_acq` takes finite differences for this model.
    """

    def __init__(self, input_dim, z_dim: int = 2, data_kernel: str = "RBF", num_latents: Optional[int] = None,
                 shared_input_space: bool = False, num_tasks: Optional[int] = None, rank: Optional[int] = None,
                 data_kernel_prior=None, nn=None, nn_prior: bool = True, guide: str = "delta", W_prior_dist=None,
                 v_prior_dist=None, task_kernel_prior=None, ctx=None, **kwargs) -> None:
        if data_kernel == "Periodic":
            raise NotImplementedError("viMTDKL takes data_kernel 'RBF' or 'Matern': the reference samples no period for "
                                      "'Periodic', so its own model fails there")
        if data_kernel not in ("RBF", "Matern"):
            raise NotImplementedError("viMTDKL takes data_kernel 'RBF' or 'Matern'")
        if data_kernel_prior is not None or task_kernel_prior is not None:
            raise NotImplementedError("data_kernel_prior / task_kernel_prior programs are not supported by viMTDKL; use "
                                      "W_prior_dist, v_prior_dist and noise_prior_dist")
        super().__init__(input_dim, z_dim, data_kernel, None, nn, nn_prior, None, guide, ctx=ctx, **kwargs)
        if shared_input_space:                                  # vi_mtdkl.py:85-91
            if num_tasks is None:
                raise ValueError("Please specify num_tasks")
        elif num_latents is None:
            raise ValueError("Please specify num_latents")
        self.num_tasks = num_tasks
        self.num_latents = num_tasks if num_latents is None else num_latents
        self.rank = rank
        self.shared_input = bool(shared_input_space)
        self.W_prior_dist = W_prior_dist
        self.v_prior_dist = v_prior_dist

    # ---- shapes and sites
    def _num_tasks(self):
        if self.num_tasks is None:                              # vi_mtdkl.py:108-109
            return len(np.unique(np.asarray(self.X_train)[:, -1]))
        return int(self.num_tasks)

    def _site_list(self):
        """(name, prior, shape) of the kernel and noise sites in the reference's order (vi_mtdkl.py:130-209)"""
        L, T, d = int(self.num_latents), self._num_tasks(), self.kernel_dim
        R = int(self.rank) if self.rank is not None else T - 1
        return [("k_length", P.LogNormal(0.0, 1.0), (L, d)), ("k_scale", P.Normal(1.0, 1e-4), (L, 1)),
                ("W", self.W_prior_dist or P.Normal(0.0, 10.0), (L, T, R)),
                ("v", self.v_prior_dist or P.LogNormal(0.0, 1.0), (L, T)),
                ("noise", self.noise_prior_dist or P.LogNormal(0.0, 1.0), (T,))]

    def _points(self, X):
        """(network inputs [n, D], int32 task ids of the GP rows, group) of an input array"""
        from .mtgp import lcm_points
        return lcm_points(self._set_data(X), self._num_tasks(), self.shared_input)

    def _mlp_inputs(self, X):
        return self._points(X)[0]

    def _theta(self, u):
        """the unconstrained vector of the kernel sites -> {name: constrained value in the site's shape}"""
        out, o = {}, 0
        for name, pr, shape in self._site_list():
            n = int(np.prod(shape))
            out[name] = np.asarray(pr.transform(u[o:o + n]), dtype=np.float64).reshape(shape)
            o += n
        return out

    def _kernel_dict(self, sites):
        return sites

    def _lcm(self, kp):
        """a kernel_params dict (one draw) -> theta [L, d+2], B [L, T, T], noise [T] of the C ABI"""
        from .mtgp import lcm_task_matrix
        L, T, d = int(self.num_latents), self._num_tasks(), self.kernel_dim
        theta = np.ones((L, d + 2))
        theta[:, :d] = np.broadcast_to(np.asarray(kp["k_length"], dtype=np.float64).reshape(L, -1), (L, d))
        theta[:, d] = np.asarray(kp["k_scale"], dtype=np.float64).reshape(L)
        B = lcm_task_matrix(np.asarray(kp["W"], dtype=np.float64).reshape(L, T, -1), np.asarray(kp["v"]).reshape(L, T))
        noise = np.broadcast_to(np.asarray(kp["noise"], dtype=np.float64).reshape(-1), (T,)).copy()
        return theta, B, noise

    # ---- fit
    def _init_params(self, rng):
        """kernel sites at their prior median, W at the median of INIT_MEDIAN_DRAWS prior draws (see the class docstring),
        then the network as viDKL"""
        u = []
        for name, pr, shape in self._site_list():
            if name == "W":
                u.append(np.asarray(pr.inverse(np.median(pr.sample(rng, (INIT_MEDIAN_DRAWS,) + shape), axis=0))).ravel())
            else:
                u.append(np.full(int(np.prod(shape)), float(pr.inverse(pr.median()))))
        return np.concatenate(u), self._init_network(rng)

    def _log_joint(self, X, Xd, yd, jitter):
        """log p(y, sites) over (u of the kernel sites, flat network parameters) and its gradient: b2gp_mtdkl_mll's
        likelihood, the sites' priors in the constrained space without the Jacobian (as viDKL), the network's prior"""
        sites = self._site_list()
        nth = sum(int(np.prod(sh)) for _, _, sh in sites)
        _, task, group = self._points(X)
        wmask = self._weight_mask()

        def f(v, jacobian=False):
            u, flat = v[:nth], v[nth:]
            kp = self._theta(u)
            theta, B, noise = self._lcm(kp)
            val, gt, gB, gn, gp, _, info = self.ctx.mtdkl_mll(self._fused, Xd, task, yd, self.widths, self.act, flat, theta, B,
                                                              noise, group, jitter)
            if info != 0 or not np.isfinite(val):
                return -np.inf, np.zeros_like(v)
            d = self.kernel_dim
            # d value / d (constrained site): the C ABI's d/dlog for lengthscales, scale and noise; B's chain rule to W, v
            g = {"k_length": gt[:, :d] / kp["k_length"], "k_scale": (gt[:, d] / theta[:, d]).reshape(-1, 1),
                 "W": np.einsum("qab,qbr->qar", gB + gB.transpose(0, 2, 1), kp["W"]), "v": np.diagonal(gB, axis1=1, axis2=2),
                 "noise": gn / noise}
            gu, o = np.zeros(nth), 0
            for name, pr, shape in sites:
                n = int(np.prod(shape))
                uk, t = u[o:o + n], kp[name].reshape(-1)
                dt = np.asarray(pr.dtheta_du(uk), dtype=np.float64)
                val += float(np.sum(pr.log_prob(t)))
                gu[o:o + n] = (g[name].reshape(-1) + pr.dlog_prob(t)) * dt
                if jacobian:
                    val += float(np.sum(pr.log_abs_jac(uk)))
                    gu[o:o + n] += pr.dlog_abs_jac(uk)
                o += n
            if self.nn_prior:
                lp, glp = _nn_log_prior(wmask, flat)
                val += lp
                gp = gp + glp
            return val, np.concatenate([gu, gp])
        return f, nth

    # ---- predict
    def _posterior_lcm(self, X_new, flat, kp, yres, noiseless, want, eps=None, jitter=1e-6):
        """the LCM posterior on the embeddings of one weight set: flat [P], kp one draw's kernel_params, yres [rows]"""
        Xtr, ttr, group = self._points(self.X_train)
        Xn, tn, _ = self._points(X_new)
        Ztr = self.ctx.mlp_forward(Xtr, self.widths, self.act, flat)[0]
        Zn = self.ctx.mlp_forward(Xn, self.widths, self.act, flat)[0]
        if group > 1:
            Ztr, Zn = np.repeat(Ztr, group, axis=0), np.repeat(Zn, group, axis=0)
        theta, B, noise = self._lcm(kp)
        return self.ctx.posterior_multitask(self._fused, Ztr, ttr, np.asarray(yres, dtype=np.float64).reshape(-1), Zn, tn,
                                            theta[None], B[None], noise[None], group, noiseless, jitter, want, eps)

    def _channels(self, nn_params, k_params):
        """[(flat, kernel_params, y)] per channel of y_train"""
        flat = self.to_flat(nn_params)
        y = np.asarray(self.y_train, dtype=np.float64)
        if y.ndim == 1:
            return [(flat, k_params, y)]
        return [(flat[c], {k: np.asarray(v)[c] for k, v in k_params.items()}, y[c]) for c in range(y.shape[0])]

    def _posterior_batched(self, X_new, params, batched, noiseless, want, eps=None, **kwargs):
        """the seam of the acquisition functions: params = (nn_params, kernel_params) of one fit; one channel"""
        nn_params, kp = params
        (flat, kpc, y), = self._channels(nn_params, kp)
        return self._posterior_lcm(X_new, flat, kpc, y, noiseless, want, eps, float(kwargs.get("jitter", 1e-6)))

    def _posterior_grad(self, X_new, params, batched, noiseless, **kwargs):
        raise NotImplementedError("multi-task models have no analytic posterior gradient; optimize_acq differences them")

    def _kg_terms(self, X_new, params, noiseless, jitter):
        """acquisition.kg's per-candidate terms of the rank-1 update (b2gp_kg_v) for one fit, multitask form.  With
        bj = jitter sum_q B_q[t, t] (the data kernel's own jitter on k_pp's diagonal, which the cross-covariance with an
        appended training row does not carry) and the noise term L (noise[t] + jitter) added once per latent:
        diag_sub = bj + L (noise_p[t] + jitter) and noise_plus_jitter = bj + L (noise[t] + jitter), t the candidate's task.
        The Kronecker form is refused: observing a point there observes all T tasks, a rank-T update (the reference's kg
        appends one y per point and fails on the P*T outputs)."""
        if self.shared_input:
            raise NotImplementedError("KG is not supported in the Kronecker form (shared_input_space=True): observing a "
                                      "point observes every task, which is not the rank-1 update KG evaluates")
        _, kp = params
        (_, kpc, _), = self._channels(params[0], kp)
        _, t, _ = self._points(X_new)
        _, B, noise = self._lcm(kpc)
        L = B.shape[0]
        bj = jitter * B[:, t, t].sum(0)
        noise_p = noise * (0.0 if noiseless else 1.0)
        return bj + L * (noise_p[t] + jitter), bj + L * (noise[t] + jitter)

    def get_mvn_posterior(self, X_new, nn_params, k_params, noiseless: bool = False, y_residual=None,
                          **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """vi_mtdkl.py:211-247: mean [P'] and covariance [P', P'] for one set of network weights and kernel parameters
        (P' = P, or P*T in the Kronecker form)"""
        y = self.y_train if y_residual is None else y_residual
        out = self._posterior_lcm(X_new, self.to_flat(nn_params), k_params, y, noiseless, ("mean", "cov"),
                                  jitter=float(kwargs.get("jitter", 1e-6)))
        return out["mean"][0], out["cov"][0]

    def predict(self, rng_key, X_new, params=None, noiseless: bool = False, *args, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """vidkl.py:277-318 with the LCM posterior: (mean, var), [P'] or, for C channels, [C, P'] (one posterior per
        channel)"""
        nn_params, k_params = (self.nn_params, self.kernel_params) if params is None else params
        X_new = self._set_data(X_new)
        res = [self._posterior_lcm(X_new, f, kp, y, noiseless, ("mean", "var"), jitter=float(kwargs.get("jitter", 1e-6)))
               for f, kp, y in self._channels(nn_params, k_params)]
        mean, var = np.stack([r["mean"][0] for r in res]), np.stack([r["var"][0] for r in res])
        if np.asarray(self.y_train).ndim == 2:
            return mean, var
        return mean[0], var[0]

    def embed(self, X_new) -> np.ndarray:
        """vidkl.py:371-384: z [N, d], or [C, N, d] with C channels.  The multitask form's task column is stripped first."""
        flat = self.to_flat(self.nn_params)
        Z = self.ctx.mlp_forward(self._points(X_new)[0], self.widths, self.act, np.atleast_2d(flat))
        return Z if flat.ndim == 2 else Z[0]
