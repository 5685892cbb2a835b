"""
utils.py -- host helpers of the reference that the posterior path touches (gpax/utils/utils.py),
restated on NumPy.  Nothing here is numerical work.
"""
import numpy as np


_X64 = False


def enable_x64():
    """gpax/utils/utils.py:19-21.  The GPU path always computes in fp64; what the switch changes here is what it
    changes in the reference's random stream: `jax.random.normal` draws float64 variates from 64-bit words instead of
    float32 ones from 32-bit words, so y_sampled for a given key follows the reference in either mode."""
    global _X64
    _X64 = True


def x64_enabled() -> bool:
    return _X64


def get_keys(seed: int = 0):
    """gpax/utils/utils.py:24-30: `jax.random.split(jax.random.PRNGKey(seed))` -- the same two uint32[2] keys
    (prng.py restates JAX's threefry key derivation)."""
    from .prng import PRNGKey, split
    k = split(PRNGKey(seed), 2)
    return k[0], k[1]


def posterior_eps(rng_key, num_draws, n, P, dtype=np.float32, per_draw_keys=True):
    """Standard normals behind y_sampled, shape (num_draws, n, P), float64.

    An int seed or a JAX-style uint32[2] key reproduces the reference's stream: one sub-key per hyper-parameter draw
    (`jra.split(rng_key, num_samples)`, gp.py:391), `jax.random.normal(key, (n, P))` in the precision the reference
    runs in (float32 unless `enable_x64()` was called, as there).  `per_draw_keys=False` is the
    single-draw `_predict` (gp.py:279-293), which hands `rng_key` to the sampler as it is.  A numpy Generator (or
    None) is this package's own extension and draws from that generator."""
    if rng_key is None or isinstance(rng_key, np.random.Generator):
        return seed_from_key(rng_key).standard_normal((num_draws, n, P))
    from . import prng
    if per_draw_keys:
        return prng.mvn_eps(rng_key, num_draws, n, P, dtype)
    return prng.normal(prng.as_key(rng_key), (n, P), dtype).astype(np.float64)[None]


def seed_from_key(rng_key):
    """Accept an int, a JAX-style uint32[2] key, a numpy Generator, or None."""
    if rng_key is None:
        return np.random.default_rng(0)
    if isinstance(rng_key, np.random.Generator):
        return rng_key
    arr = np.asarray(rng_key)
    if arr.dtype == object:
        raise TypeError("rng_key must be an int or an integer array")
    return np.random.default_rng([int(v) & 0xFFFFFFFF for v in arr.reshape(-1)])


def split_in_batches(X_new, batch_size: int = 100, dim: int = 0):
    """gpax/utils/utils.py:33-51.  Same chunks as the reference for X_new.shape[dim] >= batch_size; the
    reference raises UnboundLocalError when there are fewer rows than batch_size (SURVEY.md section 9) --
    here that case returns the single short chunk."""
    if dim not in [0, 1]:
        raise NotImplementedError("'dim' must be equal to 0 or 1")
    n = X_new.shape[dim]
    num_batches = n // batch_size
    out = []
    for i in range(num_batches):
        out.append(X_new[i * batch_size:(i + 1) * batch_size] if dim == 0 else X_new[:, i * batch_size:(i + 1) * batch_size])
    start = num_batches * batch_size
    rest = X_new[start:] if dim == 0 else X_new[:, start:]
    if rest.shape[dim] > 0:
        out.append(rest)
    return out


def initialize_inducing_points(X, ratio=0.1, method="uniform", key=None):
    """gpax/utils/utils.py:171-212.  'uniform' uses proper integer indices (the reference casts them to
    int8 and wraps beyond 127 rows, SURVEY.md section 9); 'random' draws without replacement from `key`."""
    if not 0 < ratio < 1:
        raise ValueError("The 'ratio' value must be between 0 and 1")
    X = np.asarray(X)
    n = X.shape[0]
    m = int(n * ratio)
    if method == "uniform":
        idx = np.linspace(0, n - 1, m).astype(np.int64)
        return X[idx]
    if method == "random":
        if key is None:
            raise ValueError("A random key must be provided for random selection")
        idx = seed_from_key(key).choice(n, size=m, replace=False)
        return X[idx]
    if method == "kmeans":
        from sklearn.cluster import KMeans
        return np.asarray(KMeans(n_clusters=m, random_state=0, n_init=10).fit(X).cluster_centers_)
    raise ValueError("Method must be 'uniform', 'random', or 'kmeans'")


# ---- user mean and kernel functions written with named parameters (gpax/utils/fn.py)
def _params_fn(func, leading, params_names, name=None):
    """A copy of `func` whose arguments are `leading` + `params` and whose body reads every name in `params_names` as
    params["name"].  The body is rewritten on its syntax tree and compiled in `func`'s own globals, so the modules the
    user's function refers to (np, math, ...) resolve as they did."""
    import ast
    import inspect
    import textwrap

    tree = ast.parse(textwrap.dedent(inspect.getsource(func)))
    fdef = tree.body[0]
    names = set(params_names)

    class ToParams(ast.NodeTransformer):
        def visit_Name(self, node):
            if node.id in names:
                return ast.copy_location(ast.Subscript(value=ast.Name(id="params", ctx=ast.Load()), slice=ast.Constant(node.id),
                                                       ctx=node.ctx), node)
            return node

    fdef = ToParams().visit(fdef)
    fdef.decorator_list = []
    fdef.name = name or fdef.name
    fdef.args = ast.arguments(posonlyargs=[], args=[ast.arg(arg=a) for a in list(leading) + ["params"]], vararg=None, kwonlyargs=[],
                              kw_defaults=[], kwarg=None, defaults=[])
    ns = dict(func.__globals__)
    exec(compile(ast.fix_missing_locations(tree), inspect.getsourcefile(func) or "<set_fn>", "exec"), ns)
    return ns[fdef.name]


def set_fn(func):
    """gpax/utils/fn.py set_fn: f(x, a, b, ...) -> f(x, params) reading a, b, ... from the dict `params`, the form
    ExactGP's mean_fn takes with a mean_fn_prior."""
    import inspect
    args = list(inspect.signature(func).parameters)
    return _params_fn(func, args[:1], args[1:])


def set_kernel_fn(func, independent_vars=("X", "Z"), jit_decorator=True, docstring=None):
    """gpax/utils/fn.py set_kernel_fn: k(X, Z, p1, p2, ...) -> k(X, Z, params, noise=0, jitter=1e-6, **kwargs) reading its
    parameters (the arguments without a default, other than `independent_vars`) from `params`, and adding
    (noise + jitter) I when X.shape == Z.shape -- the kernel-callable form ExactGP / viGP take.  `jit_decorator` is
    accepted for the reference's signature and ignored: there is no tracer on this side."""
    import functools
    import inspect
    sig = inspect.signature(func)
    names = [k for k, v in sig.parameters.items() if v.default is inspect.Parameter.empty and k not in independent_vars]
    core = _params_fn(func, list(independent_vars), names, name=func.__name__)

    @functools.wraps(func)
    def kernel_fn(X, Z, params, noise=0, jitter=1e-6, **kwargs):
        k = np.asarray(core(X, Z, params))
        if np.shape(X) == np.shape(Z):
            k = k + (noise + jitter) * np.eye(np.shape(X)[0])
        return k
    kernel_fn.__doc__ = docstring if docstring else func.__doc__
    del kernel_fn.__wrapped__
    return kernel_fn


def _set_noise_kernel_fn(func):
    """gpax/utils/fn.py _set_noise_kernel_fn: the kernel of a noise model, reading its "k..." parameters under
    "k_noise..." names (k_noise_length for k_length, ...).  The keys are mapped before the call rather than the
    source rewritten, so this works on any kernel callable, the fused RBFKernel / MaternKernel / PeriodicKernel included
    (their parameters are read inside the Gram build, not in Python source)."""
    import functools

    @functools.wraps(func)
    def noise_kernel_fn(X, Z, params, *args, **kwargs):
        mapped = {k: v for k, v in params.items() if not k.startswith("k")}
        mapped.update({"k" + k[len("k_noise"):]: v for k, v in params.items() if k.startswith("k_noise")})
        return func(X, Z, mapped, *args, **kwargs)
    return noise_kernel_fn
