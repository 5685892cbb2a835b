"""CPU: the log joints behind vExactGP.fit and UIGP.fit (gpax_b200/variants.py) against a SciPy restatement of the
reference models' log densities (gpax/models/vgp.py:55-121, uigp.py:78-129), on a fake context whose mll_batch runs the
NumPy oracles per member."""
import contextlib
import math

import numpy as np
import pytest
from scipy import stats

import oracle.dkl_oracle as dko
import oracle.fit_oracle as fo
from gpax_b200 import UIGP, vExactGP
from gpax_b200 import priors as P
from gpax_b200.variants import _UIGPLogJoint, _VExactLogJoint

KINDS = ["RBF", "Matern", "Periodic"]
JITTER = 1e-6


class FakeCtx:
    """Context.mll_batch on the host: oracle.fit_oracle.mll_grad and oracle.dkl_oracle.mll_dz per member"""

    def __init__(self):
        self.calls = 0

    def mll_batch(self, kind, X, yres, theta, jitter=1e-6, want_grad=True, want_alpha=False, want_grad_x=False):
        self.calls += 1
        B, N, d = X.shape
        val, grad, gx = np.zeros(B), np.zeros((B, d + 3)), np.zeros((B, N, d))
        for b in range(B):
            val[b], grad[b], _, _, _ = fo.mll_grad(kind, X[b], yres[b], theta[b], jitter)
            if want_grad_x:
                _, _, gx[b], _ = dko.mll_dz(kind, X[b], yres[b], theta[b], jitter)
        return val, grad if want_grad else None, None, gx if want_grad_x else None, np.zeros(B, dtype=np.int32)


def scipy_dist(pr):
    """the gpax_b200.priors object as a frozen SciPy distribution"""
    if isinstance(pr, P.LogNormal):
        return stats.lognorm(s=pr.scale, scale=math.exp(pr.loc))
    if isinstance(pr, P.HalfNormal):
        return stats.halfnorm(scale=pr.scale)
    raise TypeError(pr)


def scipy_gram(kind, X, ell, scale, period, noise, jitter):
    """gpax/kernels/kernels.py's three kernels written out, plus (noise + jitter) on the diagonal"""
    D = X[:, None, :] - X[None, :, :]
    if kind == "Periodic":
        K = scale * np.exp(-2.0 * ((np.sin(np.pi * D / period) / ell) ** 2).sum(-1))
    else:
        r2 = ((D / ell) ** 2).sum(-1)
        if kind == "RBF":
            K = scale * np.exp(-0.5 * r2)
        else:
            r = np.sqrt(r2 + 1e-12)
            K = scale * (1 + math.sqrt(5) * r + 5.0 / 3.0 * r2) * np.exp(-math.sqrt(5) * r)
    return K + (noise + jitter) * np.eye(len(X))


def mvn_logpdf(y, K):
    return stats.multivariate_normal(mean=np.zeros(len(y)), cov=K).logpdf(y)


def vexact_density(lj, u):
    """vgp.py:55-121 at the unconstrained point u: the B likelihoods, the site priors and log |dtheta/du| (every default
    site is positive, theta = exp(u))"""
    B, d, kind, m = lj.B, lj.d, lj.kind, lj.m
    a = 0
    ell = np.exp(u[a:a + B * d]).reshape(B, d)
    a += B * d
    scale = np.exp(u[a:a + B])
    a += B
    noise = np.exp(u[a:a + B])
    a += B
    period = np.exp(u[a:a + B]) if kind == "Periodic" else np.ones(B)
    X, y = np.asarray(m.X_train), np.asarray(m.y_train).reshape(B, -1)
    f_loc = np.zeros_like(y) if m.mean_fn is None else np.asarray(m.mean_fn(X)).reshape(B, -1)     # vgp.py:77-82
    out = sum(mvn_logpdf(y[b] - f_loc[b], scipy_gram(kind, X[b], ell[b], scale[b], period[b], noise[b], JITTER)) for b in range(B))
    out += stats.lognorm(s=1.0).logpdf(ell).sum()                                   # vgp.py:114: always LogNormal(0, 1)
    out += scipy_dist(m.lengthscale_prior_dist or P.LogNormal()).logpdf(scale).sum()  # vgp.py:116-117: k_scale's prior
    out += scipy_dist(m.noise_prior_dist or P.LogNormal()).logpdf(noise).sum()
    if kind == "Periodic":
        out += stats.lognorm(s=1.0).logpdf(period).sum()
    return out + u.sum()


def uigp_density(lj, u):
    """uigp.py:78-129 at u: sigma_x, X_prime ~ Normal(X, sigma_x), the kernel sites of gp.py:222-247, the likelihood on
    X_prime, and log |dtheta/du| of every positive site (X_prime is not transformed)"""
    N, d, kind, m = lj.N, lj.d, lj.kind, lj.m
    sx = np.exp(u[:d])
    Xp = u[d:d + N * d].reshape(N, d)
    k = u[d + N * d:]
    ell, scale = np.exp(k[:d]), math.exp(k[d])
    period = math.exp(k[d + 1]) if kind == "Periodic" else 1.0
    noise = math.exp(k[-1])
    out = mvn_logpdf(lj.y, scipy_gram(kind, Xp, ell, scale, period, noise, JITTER))
    out += scipy_dist(m.sigma_x_prior_dist or P.HalfNormal(0.1)).logpdf(sx).sum()
    out += stats.norm(loc=lj.X, scale=sx[None, :]).logpdf(Xp).sum()
    out += scipy_dist(m.lengthscale_prior_dist or P.LogNormal()).logpdf(ell).sum() + stats.lognorm(s=1.0).logpdf(scale)
    if kind == "Periodic":
        out += stats.lognorm(s=1.0).logpdf(period)
    out += scipy_dist(m.noise_prior_dist or P.LogNormal()).logpdf(noise)
    return out + u[:d].sum() + k.sum()


def vexact_model(kind, d, B, N=7, seed=0, **kw):
    rng = np.random.default_rng(seed)
    m = vExactGP(d, kind, ctx=FakeCtx(), **kw)
    X = rng.uniform(0, 1, (B, N, d))
    m.X_train, m.y_train = X, np.sin(3 * X.sum(-1)) + 0.1 * rng.standard_normal((B, N))
    return m


def uigp_model(kind, d, N=7, seed=0, **kw):
    rng = np.random.default_rng(seed)
    m = UIGP(d, kind, ctx=FakeCtx(), **kw)
    X = rng.uniform(0, 1, (N, d))
    m.X_train, m.y_train = X, np.sin(3 * X.sum(-1)) + 0.1 * rng.standard_normal(N)
    return m


def check_value_and_grad(lj, density, u):
    val, grad = lj(u, jacobian=True)
    assert val == pytest.approx(density(lj, u), rel=1e-10, abs=1e-10)
    h = 1e-5
    fd = np.array([(density(lj, u + h * e) - density(lj, u - h * e)) / (2 * h) for e in np.eye(lj.dim)])
    assert np.max(np.abs(grad - fd)) <= 1e-6 * max(1.0, np.max(np.abs(fd)))


VPRIORS = [{}, {"lengthscale_prior_dist": P.LogNormal(0.5, 0.7)}, {"noise_prior_dist": P.HalfNormal(2.0)},
           {"mean_fn": lambda X: 0.5 * X.sum(-1, keepdims=True) - 0.2}]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("kw", VPRIORS, ids=["default", "lengthscale_prior", "noise_prior", "mean_fn"])
def test_vexact_log_joint_matches_the_reference_density(kind, d, B, kw):
    lj = _VExactLogJoint(vexact_model(kind, d, B, **kw), JITTER)
    u = lj.init_u() + 0.3 * np.random.default_rng(1).standard_normal(lj.dim)
    check_value_and_grad(lj, vexact_density, u)
    assert lj.m.ctx.calls == 1                     # one mll_batch call per evaluation, whatever B


UPRIORS = [{}, {"lengthscale_prior_dist": P.LogNormal(0.5, 0.7)}, {"noise_prior_dist": P.HalfNormal(2.0)},
           {"sigma_x_prior_dist": P.HalfNormal(0.3)}]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("kw", UPRIORS, ids=["default", "lengthscale_prior", "noise_prior", "sigma_x_prior"])
def test_uigp_log_joint_matches_the_reference_density(kind, d, kw):
    lj = _UIGPLogJoint(uigp_model(kind, d, **kw), JITTER)
    rng = np.random.default_rng(2)
    u = lj.init_u() + 0.05 * rng.standard_normal(lj.dim)
    check_value_and_grad(lj, uigp_density, u)


def test_uigp_starts_at_the_observed_inputs_and_prior_medians():
    lj = _UIGPLogJoint(uigp_model("RBF", 2), JITTER)
    sx, Xp, th = lj._split(lj.init_u())
    np.testing.assert_allclose(sx, 0.6744897501960817 * 0.1)
    np.testing.assert_array_equal(Xp, lj.X)
    np.testing.assert_allclose(th[:4], 1.0)


def test_vgp_lengthscale_prior_moves_only_the_k_scale_term():
    """vgp.py:101-121 samples k_length from LogNormal(0, 1) always and hands `lengthscale_prior_dist` to k_scale; the
    wiring is kept as the reference writes it"""
    pr = P.LogNormal(0.5, 0.7)
    a = _VExactLogJoint(vexact_model("RBF", 2, 3), JITTER)
    b = _VExactLogJoint(vexact_model("RBF", 2, 3, lengthscale_prior_dist=pr), JITTER)
    u = np.random.default_rng(3).standard_normal(a.dim)
    u[6:9] = 0.2                                   # the k_scale block
    (va, ga), (vb, gb) = a(u, True), b(u, True)
    t = np.exp(u[6:9])
    assert vb - va == pytest.approx(float(np.sum(pr.log_prob(t) - P.LogNormal().log_prob(t))), rel=1e-12)
    keep = np.r_[0:6, 9:a.dim]
    np.testing.assert_array_equal(ga[keep], gb[keep])
    assert not np.allclose(ga[6:9], gb[6:9])


def test_vexact_sample_shapes_and_a_short_run():
    m = vexact_model("Periodic", 2, 3)
    lj = _VExactLogJoint(m, JITTER)
    s = lj.to_dict(np.stack([lj.init_u()] * 4))
    assert s["k_length"].shape == (4, 3, 2) and s["k_scale"].shape == (4, 3)
    assert s["noise"].shape == (4, 3) and s["period"].shape == (4, 3)
    m.fit(0, m.X_train, m.y_train, num_warmup=30, num_samples=30, num_chains=2, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert s["k_length"].shape == (60, 3, 2) and s["k_scale"].shape == (60, 3) and s["noise"].shape == (60, 3)
    assert all(np.isfinite(v).all() for v in s.values())
    assert m.get_samples(chain_dim=True)["k_length"].shape == (2, 30, 3, 2)


def test_uigp_sample_shapes_and_a_short_run():
    m = uigp_model("RBF", 2, N=6)
    with pytest.warns(UserWarning):
        m.fit(0, m.X_train, m.y_train, num_warmup=30, num_samples=30, progress_bar=False, print_summary=False)
    s = m.get_samples()
    assert s["sigma_x"].shape == (30, 2) and s["X_prime"].shape == (30, 6, 2) and s["k_length"].shape == (30, 2)
    assert s["k_scale"].shape == (30,) and s["noise"].shape == (30,)
    assert all(np.isfinite(v).all() for v in s.values())


def test_uigp_summary_leaves_out_x_prime(capsys):
    m = uigp_model("RBF", 1, N=5)
    lj = _UIGPLogJoint(m, JITTER)

    class R:
        def get_samples(self, group_by_chain=False):
            return {k: v[None] for k, v in lj.to_dict(np.stack([lj.init_u()] * 3)).items()}
    m.mcmc = R()
    m._print_summary()
    out = capsys.readouterr().out
    assert "sigma_x" in out and "k_length" in out and "X_prime" not in out


def _prog():
    return {}


@pytest.mark.parametrize("kw, what", [({"kernel_prior": _prog}, "kernel_prior"), ({"noise_prior": _prog}, "noise_prior"),
                                      ({"mean_fn": lambda x: 0 * x[..., 0], "mean_fn_prior": _prog}, "mean_fn_prior")])
def test_vexact_refusals(kw, what):
    with pytest.warns((UserWarning, FutureWarning)) if what != "mean_fn_prior" else contextlib.nullcontext():
        m = vexact_model("RBF", 1, 2, **kw)
    with pytest.raises(NotImplementedError, match=what):
        _VExactLogJoint(m, JITTER)


def test_vexact_refuses_callable_kernels_and_foreign_priors():
    m = vExactGP(1, lambda X, Z, p, noise=0, jitter=1e-6: np.eye(len(X)), ctx=FakeCtx())
    m.X_train, m.y_train = np.zeros((2, 3, 1)), np.zeros((2, 3))
    with pytest.raises(NotImplementedError, match="callable kernels"):
        _VExactLogJoint(m, JITTER)
    with pytest.raises(TypeError):
        _VExactLogJoint(vexact_model("RBF", 1, 2, noise_prior_dist=object()), JITTER)


@pytest.mark.parametrize("kw, what", [({"kernel_prior": _prog}, "kernel_prior"), ({"mean_fn": lambda x: 0 * x[:, 0]}, "mean functions"),
                                      ({"mean_fn": lambda x, p: 0 * x[:, 0], "mean_fn_prior": _prog}, "mean functions")])
def test_uigp_refusals(kw, what):
    with pytest.warns(UserWarning) if "kernel_prior" in kw else contextlib.nullcontext():
        m = uigp_model("RBF", 1, **kw)
    with pytest.raises(NotImplementedError, match=what):
        _UIGPLogJoint(m, JITTER)


def test_uigp_refuses_callable_kernels_and_foreign_priors():
    m = UIGP(1, lambda X, Z, p, noise=0, jitter=1e-6: np.eye(len(X)), ctx=FakeCtx())
    m.X_train, m.y_train = np.zeros((3, 1)), np.zeros(3)
    with pytest.raises(NotImplementedError, match="callable kernels"):
        _UIGPLogJoint(m, JITTER)
    with pytest.raises(TypeError):
        _UIGPLogJoint(uigp_model("RBF", 1, sigma_x_prior_dist=object()), JITTER)


def test_vexact_predict_in_batches_splits_the_point_axis():
    m = vexact_model("RBF", 1, 3)
    seen = []

    def fn(Xi):
        seen.append(Xi.shape)
        return np.ones((3, Xi.shape[1])), np.ones((5, 2, 3, Xi.shape[1]))
    mean, ys = m.predict_in_batches(0, np.zeros((3, 10)), batch_size=4, predict_fn=fn)
    assert seen == [(3, 4, 1), (3, 4, 1), (3, 2, 1)]
    assert mean.shape == (3, 10) and ys.shape == (5, 2, 3, 10)
