"""CPU: the log joints behind VarNoiseGP.fit and MeasuredNoiseGP.fit with prior programs and noise mean functions
(gpax_b200/variants.py, inference.ProgramLogJoint with a fixed noise vector) against a SciPy restatement of the reference
models (gpax/models/hskgp.py:105-149, mngp.py:75-97), on a fake context whose likelihoods run the NumPy oracles."""
import math

import numpy as np
import pytest
from scipy import stats

import oracle.fit_oracle as fo
import oracle.gp_oracle as go
from gpax_b200 import MeasuredNoiseGP, VarNoiseGP
from gpax_b200 import priors as P
from gpax_b200.inference import ProgramLogJoint
from gpax_b200.variants import _VarNoiseLogJoint, _VarNoiseProgramLogJoint

JITTER = 1e-6
N = 7


class FakeCtx:
    """Context.mll / mll_draws / mll_draws_v / posterior on the host (oracle.fit_oracle, oracle.gp_oracle)"""

    def __init__(self):
        self.calls = {"mll": 0, "mll_draws": 0, "mll_draws_v": 0}

    def _one(self, kind, X, yres, theta, jitter, noise_vec):
        """(value, grad, alpha, grad_noise_vec, info); a failed factorisation gives NaN and info 1, as the library does"""
        try:
            val, grad, alpha, gnv, _ = fo.mll_grad(kind, X, yres, theta, jitter, noise_vec)
            return val, grad, alpha, np.zeros(len(X)) if gnv is None else gnv, 0
        except (np.linalg.LinAlgError, ValueError):
            nan = np.full(len(X), np.nan)
            return np.nan, np.full(X.shape[1] + 3, np.nan), nan, nan, 1

    def mll(self, kind, X, yres, theta, jitter=1e-6, want_grad=True, want_alpha=False, noise_vec=None):
        self.calls["mll"] += 1
        val, grad, alpha, gnv, info = self._one(kind, X, yres, theta, jitter, noise_vec)
        out = (val, grad if want_grad else None, alpha if want_alpha else None, info)
        return out if noise_vec is None else out + (gnv if want_grad else None,)

    def mll_draws(self, kind, X, yres, theta, jitter=1e-6, want_grad=True, want_alpha=False):
        self.calls["mll_draws"] += 1
        S = len(theta)
        Y = np.broadcast_to(yres, (S, len(X)))
        rows = [self._one(kind, X, Y[s], theta[s], jitter, None) for s in range(S)]
        return (np.array([r[0] for r in rows]), np.stack([r[1] for r in rows]) if want_grad else None,
                np.stack([r[2] for r in rows]) if want_alpha else None, np.array([r[4] for r in rows], dtype=np.int32))

    def mll_draws_v(self, kind, X, yres, theta, noise_vec, jitter=1e-6, want_grad=True, want_alpha=False):
        self.calls["mll_draws_v"] += 1
        S = len(theta)
        Y, NV = np.broadcast_to(yres, (S, len(X))), np.broadcast_to(noise_vec, (S, len(X)))
        rows = [self._one(kind, X, Y[s], theta[s], jitter, NV[s]) for s in range(S)]
        return (np.array([r[0] for r in rows]), np.stack([r[1] for r in rows]) if want_grad else None,
                np.stack([r[2] for r in rows]) if want_alpha else None, np.stack([r[3] for r in rows]) if want_grad else None,
                np.array([r[4] for r in rows], dtype=np.int32))

    def posterior(self, kind, X, yres, Xn, theta, noiseless, jitter, want, eps=None):
        d = X.shape[1]
        Y = np.broadcast_to(yres, (len(theta), len(X)))
        means, covs = [], []
        for s, th in enumerate(theta):
            params = {"k_length": th[:d], "k_scale": th[d], "noise": th[d + 1], "period": th[d + 2]}
            mu, cov = go.exact_posterior(X, Y[s], Xn, params, kind, noiseless=noiseless, jitter=jitter)
            means.append(mu)
            covs.append(cov)
        return {"mean": np.stack(means), "cov": np.stack(covs), "var": None, "y_sampled": None,
                "info": np.zeros(len(theta), dtype=np.int32)}


# ---------------------------------------------------------------------------------------------- the reference's programs
def noise_fn(x, params):                                    # tests/test_hskgp.py of the reference
    return params["a"] + params["b"] * x


def noise_fn_prior():
    return {"a": P.sample("a", P.Normal(0, 1)), "b": P.sample("b", P.Normal(0, 1))}


def mean_fn(x, params):
    return params["c"] * x ** 2


def mean_fn_prior():
    return {"c": P.sample("c", P.LogNormal(-0.7, 0.5))}


def kernel_prior():
    return {"k_length": P.sample("k_length", P.Gamma(2.0, 2.0)), "k_scale": P.sample("k_scale", P.HalfNormal(5.0))}


def noise_kernel_prior():
    return {"k_noise_length": P.sample("k_noise_length", P.LogNormal(0.3, 0.5)),
            "k_noise_scale": P.sample("k_noise_scale", P.Gamma(3.0, 2.0))}


def default_kernel_prior():                                 # the default sites of gp.py:229-247, restated
    with P.plate("ard", 1):
        ell = P.sample("k_length", P.LogNormal(0.0, 1.0))
    return {"k_length": ell, "k_scale": P.sample("k_scale", P.LogNormal(0.0, 1.0))}


def default_noise_kernel_prior():                           # hskgp.py:151-163, restated
    return {"k_noise_scale": P.sample("k_noise_scale", P.LogNormal(0.0, 1.0)),
            "k_noise_length": P.sample("k_noise_length", P.LogNormal(0.0, 1.0))}


def data(seed=0):
    rng = np.random.default_rng(seed)
    X = np.linspace(1, 2, N) + 0.05 * rng.standard_normal(N)
    return X, 0.5 * X ** 2 + (0.1 + 0.3 * (X - 1)) * rng.standard_normal(N)


def var_noise(kind="RBF", **kw):
    m = VarNoiseGP(1, kind, ctx=FakeCtx(), **kw)
    m.X_train, m.y_train = data()
    return m


# ---------------------------------------------------------------------------------------------- SciPy restatement
def gram(kind, X, ell, scale, period=1.0):
    D = X[:, None] - X[None, :]
    if kind == "Periodic":
        return scale * np.exp(-2.0 * (np.sin(np.pi * D / period) / ell) ** 2)
    return scale * np.exp(-0.5 * (D / ell) ** 2)


def mvn(x, mean, K):
    return stats.multivariate_normal(mean=mean, cov=K).logpdf(x)


# per configuration: the layout of u as (name, scipy density or None for a real site, size); "lv" is log_var
def lognorm(loc, s):
    return stats.lognorm(s=s, scale=math.exp(loc))


LN = lognorm(0.0, 1.0)
CONFIGS = {
    "noise_mean_fixed": (dict(noise_mean_fn=lambda x: 0.2 + 0.1 * x),
                         [("k_length", LN), ("k_scale", LN), ("k_noise_length", LN), ("k_noise_scale", LN), ("lv", None)]),
    "noise_mean_prior": (dict(noise_mean_fn=noise_fn, noise_mean_fn_prior=noise_fn_prior),
                         [("k_noise_scale", LN), ("k_noise_length", LN), ("a", stats.norm()), ("b", stats.norm()), ("lv", None),
                          ("k_length", LN), ("k_scale", LN)]),
    "noise_and_mean_prior": (dict(noise_mean_fn=noise_fn, noise_mean_fn_prior=noise_fn_prior, mean_fn=mean_fn,
                                  mean_fn_prior=mean_fn_prior),
                             [("k_noise_scale", LN), ("k_noise_length", LN), ("a", stats.norm()), ("b", stats.norm()),
                              ("lv", None), ("k_length", LN), ("k_scale", LN), ("c", lognorm(-0.7, 0.5))]),
    "mean_fn_prior": (dict(mean_fn=mean_fn, mean_fn_prior=mean_fn_prior),
                      [("k_noise_scale", LN), ("k_noise_length", LN), ("lv", None), ("k_length", LN), ("k_scale", LN),
                       ("c", lognorm(-0.7, 0.5))]),
    "kernel_prior": (dict(kernel_prior=kernel_prior),
                     [("k_noise_scale", LN), ("k_noise_length", LN), ("lv", None), ("k_length", stats.gamma(2.0, scale=0.5)),
                      ("k_scale", stats.halfnorm(scale=5.0))]),
    "noise_kernel_prior": (dict(noise_kernel_prior=noise_kernel_prior),
                           [("k_noise_length", lognorm(0.3, 0.5)), ("k_noise_scale", stats.gamma(3.0, scale=0.5)),
                            ("lv", None), ("k_length", LN), ("k_scale", LN)]),
    "periodic_noise_kernel_prior": (dict(noise_kernel_prior=noise_kernel_prior),
                                    [("k_noise_length", lognorm(0.3, 0.5)), ("k_noise_scale", stats.gamma(3.0, scale=0.5)),
                                     ("lv", None), ("k_length", LN), ("k_scale", LN), ("period", LN)]),
}


def split(layout, u):
    vals, o = {}, 0
    for name, _ in layout:
        size = N if name == "lv" else 1
        vals[name] = u[o:o + size] if name == "lv" else u[o]
        o += size
    return vals


def density(config, u):
    """hskgp.py:105-149 at u: both multivariate normals, the site densities and log |d site / du| of the positive sites"""
    kw, layout = CONFIGS[config]
    kind = "Periodic" if config.startswith("periodic") else "RBF"
    X, y = data()
    v = split(layout, u)
    out = 0.0
    pos = {}
    for name, dist in layout:
        if name == "lv":
            continue
        if dist.support()[0] == -np.inf:        # a real site
            pos[name] = v[name]
            out += dist.logpdf(v[name])
        else:
            pos[name] = math.exp(v[name])
            out += dist.logpdf(pos[name]) + v[name]
    mu_n = np.zeros(N)
    if "noise_mean_fn" in kw:
        f = kw["noise_mean_fn"]
        mu_n = np.log(f(X, {"a": pos["a"], "b": pos["b"]}) if "a" in pos else f(X))
    m = mean_fn(X, {"c": pos["c"]}) if "c" in pos else 0.0
    Kn = gram("RBF", X, pos["k_noise_length"], pos["k_noise_scale"]) + JITTER * np.eye(N)
    K = gram(kind, X, pos["k_length"], pos["k_scale"], pos.get("period", 1.0)) + JITTER * np.eye(N) + np.diag(np.exp(v["lv"]))
    return out + mvn(v["lv"], mu_n, Kn) + mvn(y - m, np.zeros(N), K)


def model_for(config):
    kw, _ = CONFIGS[config]
    return var_noise("Periodic" if config.startswith("periodic") else "RBF", **kw)


def point(config, seed=1):
    """a valid unconstrained point: log_var near log 0.5, a noise mean a + b x > 0"""
    _, layout = CONFIGS[config]
    rng = np.random.default_rng(seed)
    u = []
    for name, _ in layout:
        if name == "lv":
            u.extend(np.log(0.5) + 0.3 * rng.standard_normal(N))
        elif name in ("a", "b"):
            u.append(0.5 + 0.2 * rng.random())
        elif name in ("k_length", "k_noise_length"):       # well-conditioned Gram matrices on the 7 points
            u.append(math.log(0.15) + 0.1 * rng.standard_normal())
        elif name == "c":
            u.append(math.log(0.5) + 0.1 * rng.standard_normal())
        else:
            u.append(-0.3 + 0.4 * rng.standard_normal())
    return np.array(u)


def log_joint(m):
    if any(getattr(m, k) is not None for k in ("kernel_prior", "noise_kernel_prior", "noise_mean_fn_prior")) or \
            m.mean_fn_prior is not None:
        return _VarNoiseProgramLogJoint(m, JITTER)
    return _VarNoiseLogJoint(m, JITTER)


def check_value_and_grad(lj, dens, u):
    val, grad = lj(u, jacobian=True)
    assert val == pytest.approx(dens(u), rel=1e-10, abs=1e-10)
    h = 1e-5
    fd = np.array([(dens(u + h * e) - dens(u - h * e)) / (2 * h) for e in np.eye(lj.dim)])
    assert np.max(np.abs(grad - fd)) <= 1e-6 * max(1.0, np.max(np.abs(fd)))


# ---------------------------------------------------------------------------------------------- VarNoiseGP
@pytest.mark.parametrize("config", list(CONFIGS))
def test_value_and_gradient_match_the_restatement(config):
    m = model_for(config)
    lj = log_joint(m)
    assert isinstance(lj, _VarNoiseLogJoint if config == "noise_mean_fixed" else _VarNoiseProgramLogJoint)
    for seed in (1, 2):
        check_value_and_grad(lj, lambda u: density(config, u), point(config, seed))


def test_restated_default_priors_give_the_default_route():
    d_lj = _VarNoiseLogJoint(var_noise(), JITTER)
    p_lj = _VarNoiseProgramLogJoint(var_noise(kernel_prior=default_kernel_prior, noise_kernel_prior=default_noise_kernel_prior),
                                    JITTER)
    u = point("kernel_prior")                               # [ns, nl, lv, ell, scale]
    ud = np.concatenate([u[-2:], [u[1], u[0]], u[2:2 + N]])  # [ell, scale, nl, ns, lv]
    for jac in (True, False):
        vp, gp = p_lj(u, jac)
        vd, gd = d_lj(ud, jac)
        assert vp == pytest.approx(vd, rel=1e-12)
        np.testing.assert_allclose(gp[2:2 + N], gd[4:], rtol=1e-12)
        np.testing.assert_allclose(gp[[N + 2, N + 3, 1, 0]], gd[:4], rtol=1e-7)


@pytest.mark.parametrize("config", ["noise_mean_fixed", "noise_and_mean_prior", "kernel_prior"])
def test_batch_rows_are_the_single_calls(config):
    m = model_for(config)
    lj = log_joint(m)
    U = np.stack([point(config, s) for s in range(4)])
    U[2, :] = -50.0 if config != "noise_mean_fixed" else U[2, :]        # an invalid row where the programs allow one
    vals, grads = lj.batch(U, True)
    assert m.ctx.calls["mll_draws"] == 1 and m.ctx.calls["mll_draws_v"] == 1 and m.ctx.calls["mll"] == 0
    for r, u in enumerate(U):
        v, g = lj(u, True)
        assert vals[r] == v and np.array_equal(grads[r], g)


def test_to_dict_sites_in_the_reference_order():
    lj = _VarNoiseProgramLogJoint(model_for("noise_and_mean_prior"), JITTER)
    U = np.stack([point("noise_and_mean_prior", s) for s in range(3)])
    out = lj.to_dict(U)
    assert list(out) == ["k_noise_scale", "k_noise_length", "a", "b", "log_var", "k_length", "k_scale", "c", "noise"]
    assert out["log_var"].shape == (3, N) and out["k_length"].shape == (3, 1) and out["a"].shape == (3,)
    assert np.array_equal(out["log_var"], U[:, 4:4 + N]) and (out["noise"] == 0).all()
    lj = _VarNoiseProgramLogJoint(model_for("periodic_noise_kernel_prior"), JITTER)
    assert list(lj.to_dict(point("periodic_noise_kernel_prior"))) == ["k_noise_length", "k_noise_scale", "log_var", "k_length",
                                                                       "k_scale", "period", "noise"]


def test_init_falls_back_when_the_noise_mean_is_zero_at_the_medians():
    lj = _VarNoiseProgramLogJoint(model_for("noise_mean_prior"), JITTER)
    u0 = lj.init_u()                                        # a = b = 0 at the medians: log 0
    v, _ = lj(u0, True)
    assert np.isfinite(v) and np.array_equal(lj.init_u(), u0)
    assert np.array_equal(_VarNoiseProgramLogJoint(model_for("noise_mean_prior"), JITTER).init_u(), u0)   # fixed seed
    bad = point("noise_mean_prior")
    bad[2], bad[3] = -5.0, 0.0                              # a + b x < 0
    v, g = lj(bad, True)
    assert v == -np.inf and not g.any()
    lj0 = _VarNoiseProgramLogJoint(model_for("kernel_prior"), JITTER)
    assert np.isfinite(lj0(lj0.init_u(), True)[0])          # valid at the medians: no fallback


def test_per_draw_noise_mean_in_the_posterior():
    m = model_for("noise_mean_prior")
    lj = _VarNoiseProgramLogJoint(m, JITTER)
    U = np.stack([point("noise_mean_prior", s) for s in range(3)])
    samples = lj.to_dict(U)
    Xn = np.linspace(0.9, 2.1, 5)
    out, pv = m._both_posteriors(Xn, samples, True, ("mean", "cov"))
    for s in range(3):
        one = {k: np.asarray(v)[s] for k, v in samples.items()}
        o1, pv1 = m._both_posteriors(Xn, one, False, ("mean", "cov"))
        np.testing.assert_allclose(pv[s], pv1[0], rtol=1e-12)
        np.testing.assert_allclose(out["mean"][s], o1["mean"][0], rtol=1e-12)
        # against the oracle restated with the noise mean (hskgp.py:185-200)
        X = m._train_arrays()[0]
        nparams = {"k_length": one["k_noise_length"], "k_scale": one["k_noise_scale"], "noise": 0.0}
        mu, _ = go.exact_posterior(X, one["log_var"] - np.log(noise_fn(X[:, 0], one)), Xn, nparams, "RBF", noiseless=True,
                                   jitter=JITTER)
        np.testing.assert_allclose(pv[s], np.exp(mu + np.log(noise_fn(Xn, one))), rtol=1e-9)


# ---------------------------------------------------------------------------------------------- MeasuredNoiseGP
def measured(**kw):
    m = MeasuredNoiseGP(1, "RBF", ctx=FakeCtx(), **kw)
    X, y = data()
    m.X_train, m.y_train = X, y
    return m, np.linspace(0.05, 0.3, N)


def test_measured_noise_programs_match_the_restatement():
    m, nv = measured(kernel_prior=kernel_prior, mean_fn=mean_fn, mean_fn_prior=mean_fn_prior)
    lj = ProgramLogJoint(m, JITTER, noise_vec=nv)
    assert [s.name for s in lj.sites] == ["k_length", "k_scale", "c"]
    X, y = data()

    def dens(u):                                            # mngp.py:75-97
        ell, sc, c = math.exp(u[0]), math.exp(u[1]), math.exp(u[2])
        K = gram("RBF", X, ell, sc) + JITTER * np.eye(N) + np.diag(nv)
        return (mvn(y - c * X ** 2, np.zeros(N), K) + stats.gamma(2.0, scale=0.5).logpdf(ell) + stats.halfnorm(scale=5.0).logpdf(sc)
                + lognorm(-0.7, 0.5).logpdf(c) + u.sum())

    u = np.array([-0.4, 0.2, math.log(0.45)])
    check_value_and_grad(lj, dens, u)
    U = np.stack([u, u + 0.1, u - 0.2])
    vals, grads = lj.batch(U, True)
    assert m.ctx.calls["mll_draws_v"] == 1 and m.ctx.calls["mll_draws"] == 0
    for r in range(3):
        v, g = lj(U[r], True)
        assert vals[r] == v and np.array_equal(grads[r], g)
    out = lj.to_dict(U)
    assert list(out) == ["k_length", "k_scale", "c", "noise"] and (out["noise"] == 0).all()


def test_measured_noise_default_route_batch():
    from gpax_b200.variants import _MeasuredNoiseLogJoint
    m, nv = measured()
    lj = _MeasuredNoiseLogJoint(m, nv, JITTER)
    U = np.array([[-0.2, 0.1], [0.3, -0.4]])
    vals, grads = lj.batch(U, True)
    assert m.ctx.calls["mll_draws_v"] == 1
    for r in range(2):
        v, g = lj(U[r], True)
        assert vals[r] == v and np.array_equal(grads[r], g)
