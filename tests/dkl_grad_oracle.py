"""dkl_grad_oracle.py -- TEST INFRASTRUCTURE ONLY: NumPy restatement of the derivative jax.grad takes through a deep kernel
learning model in the reference's optimize_acq (gpax/acquisition/optimize.py:70-88 on viDKL / DKL): the exact-GP posterior
mean and variance on the embedding z = MLP(x), differentiated w.r.t. the RAW test input x.

  posterior_grad   dkl_oracle.mlp_forward on both input sets, grad_oracle.posterior_grad on the embeddings, then the
                   network's vector-Jacobian product back to the inputs:
                       G = d/dz,  G <- (G W_l^T) * act'(H_l) for l = L-1 .. 1,  d/dx = G W_0^T
                   act' from the post-activation as jax.nn.relu's derivative (0 at 0) and tanh's 1 - h^2

Pinned on the CPU by central differences of dkl_oracle.posterior (tests/test_dkl_posterior_grad_cpu.py)."""
import numpy as np

from oracle import dkl_oracle as dko
from oracle import grad_oracle as gro


def input_vjp(Hn, layers, act, G):
    """d/dx [P, D] of a cotangent G [P, d] at the embedding, through the stored activations Hn = mlp_forward(X_new)"""
    G = np.asarray(G, dtype=np.float64)
    for l in range(len(layers) - 1, -1, -1):
        W, _ = layers[l]
        G = G @ np.asarray(W, dtype=np.float64).T
        if l > 0:
            G = G * dko._act_grad(Hn[l], act)
    return G


def posterior_grad(kind, X, y, X_new, layers, act, params, noiseless=False, jitter=1e-6):
    """(mean [P], var [P], dmean [P, D], dvar [P, D]) of the exact GP on the embeddings, w.r.t. each raw test point"""
    z = dko.mlp_forward(X, layers, act)[-1]
    Hn = dko.mlp_forward(X_new, layers, act)
    mean, var, dmz, dvz = gro.posterior_grad(z, y, Hn[-1], params, kind, noiseless, jitter)
    return mean, var, input_vjp(Hn, layers, act, dmz), input_vjp(Hn, layers, act, dvz)
