"""The digit-plane (Ozaki) GEMM restated in NumPy (oracle/ozaki_oracle.py): the claims DESIGN.md 4.6 makes about the
int8 wgmma path, checked in exact arithmetic on the CPU, and the kernel itself checked against the restatement."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import ozaki_oracle as oz


def _rows(rng, m, k):
    return rng.standard_normal((m, k)) * np.exp(rng.normal(0, 2, (m, 1)))      # rows of very different scale


def test_digits_are_int8_and_reconstruct_to_half_a_unit_of_the_last_digit():
    rng = np.random.default_rng(0)
    A = _rows(rng, 7, 50)
    A[3] = 0.0                                                      # an all-zero row keeps exponent 0
    A[5, 0] = -A[5].__abs__().max() * 1.0                           # the row maximum itself, negative
    A[6, 1] = A[6].__abs__().max() * (1.0 - 2.0 ** -52)             # ... and one just below the next power of two
    for S in (6, 7):
        planes, scale = oz.slice_rows(A, S)
        assert planes.min() >= -128 and planes.max() <= 127         # base-256 digits in two's-complement style: int8
        assert np.abs(planes[0]).max() <= 65                        # the leading digit carries 6 bits (+ a carry)
        for i in range(A.shape[0]):
            for j in range(0, A.shape[1], 7):
                exact = Fraction(float(A[i, j]))
                got = sum(Fraction(int(planes[p, i, j]), 2 ** (6 + 8 * p)) for p in range(S)) * Fraction(float(scale[i]))
                assert abs(exact - got) <= Fraction(float(scale[i])) / 2 ** (6 + 8 * (S - 1) + 1)    # half a unit of the last digit
    assert scale[3] == 1.0


def test_class_sums_are_exact_integers_within_int32():
    rng = np.random.default_rng(1)
    A, B = _rows(rng, 5, 300), _rows(rng, 4, 300)
    PA, _ = oz.slice_rows(A, 7)
    PB, _ = oz.slice_rows(B, 7)
    D = oz.class_sums(PA, PB)
    for t in (0, 3, 6):
        ref = sum(int(PA[p, 2, kk]) * int(PB[t - p, 1, kk]) for p in range(t + 1) for kk in range(300))
        assert int(D[t, 2, 1]) == ref
    assert np.abs(D).max() < 2 ** 31
    # S pairs per class, k at the per-launch limit, digits at -128: the int32 bound behind OZ_K_MAX in ozaki.cuh
    assert 7 * oz.K_MAX * 128 * 128 < 2 ** 31


def test_long_k_is_split_into_launches_within_the_int32_bound():
    rng = np.random.default_rng(5)
    A, B, C = _rows(rng, 3, oz.K_MAX + 700), _rows(rng, 2, oz.K_MAX + 700), rng.standard_normal((3, 2))
    out = oz.gemm_nt(A, B, C, alpha=-1.0, S=7)
    ref = C - A @ B.T
    scale = np.linalg.norm(A, axis=1)[:, None] * np.linalg.norm(B, axis=1)[None, :]
    assert (np.abs(out - ref) / scale).max() < 1e-13


@pytest.mark.parametrize("S,bound", [(7, 2.0 ** -49), (6, 2.0 ** -42)])
def test_gemm_error_against_exact_rational(S, bound):
    rng = np.random.default_rng(2)
    m, n, k = 6, 5, 96
    A, B, C = _rows(rng, m, k), _rows(rng, n, k), rng.standard_normal((m, n))
    out = oz.gemm_nt(A, B, C, alpha=-1.0, S=S)
    for i in range(m):
        for j in range(n):
            exact = Fraction(float(C[i, j])) - sum(Fraction(float(A[i, kk])) * Fraction(float(B[j, kk])) for kk in range(k))
            scale = float(np.linalg.norm(A[i]) * np.linalg.norm(B[j]) + abs(C[i, j]))
            assert abs(float(Fraction(float(out[i, j])) - exact)) <= bound * scale
    low = oz.gemm_nt(A[:5], A[:5], C[:5, :5], alpha=-1.0, S=S, lower_only=True)
    full = oz.gemm_nt(A[:5], A[:5], C[:5, :5], alpha=-1.0, S=S)
    np.testing.assert_array_equal(np.tril(low), np.tril(full))
    np.testing.assert_array_equal(np.triu(low, 1), np.triu(C[:5, :5], 1))


@pytest.mark.parametrize("S", [7, 6])
def test_lower_only_trapezoid_rule(S):
    """lower_only with more rows than columns (right-hand-side rows riding below the matrix): rows < n take j <= i, the rows
    below take all n columns; everything written equals the full product, everything else is C untouched"""
    rng = np.random.default_rng(7)
    m, n, k = 9, 5, 40
    A, C = _rows(rng, m, k), rng.standard_normal((m, n))
    full = oz.gemm_nt(A, A[:n], C, alpha=-1.0, S=S)
    trap = oz.gemm_nt(A, A[:n], C, alpha=-1.0, S=S, lower_only=True)
    for i in range(m):
        for j in range(n):
            assert trap[i, j] == (full[i, j] if (i >= n or j <= i) else C[i, j]), (i, j)
    ref = C - A @ A[:n].T                                           # and the written part is the product, by plain NumPy
    written = np.tril(np.ones((m, n), bool))
    scale = np.linalg.norm(A, axis=1)[:, None] * np.linalg.norm(A[:n], axis=1)[None, :] + np.abs(C)
    assert (np.abs(trap - ref) / scale)[written].max() < (2.0 ** -49 if S == 7 else 2.0 ** -42)
    with pytest.raises(ValueError):
        oz.gemm_nt(A[:n - 1], A[:n], C[:n - 1], alpha=-1.0, S=S, lower_only=True)     # fewer rows than columns


@pytest.mark.gpu
@pytest.mark.parametrize("S", [7, 6])
def test_int8_kernel_equals_the_restatement_bit_for_bit(S):
    """exact integer products + the same fixed-order fp64 recombination on both sides -> identical doubles"""
    import gpax_b200
    ctx = gpax_b200.default_context()
    rng = np.random.default_rng(3)
    m, n, k = 1536, 1280, 544                                       # >= 132 tiles of 128 x 64 (one per SM of an H100 SXM), k >= 512, ragged k-block
    A, B, C = _rows(rng, m, k), _rows(rng, n, k), rng.standard_normal((m, n))
    before = ctx.path_counts()["oz_mma"]
    with ctx.options(ozaki=S):
        got = ctx.gemm_nt(A, B, C, alpha=-1.0, beta=1.0)
    assert ctx.path_counts()["oz_mma"] == before + 1                # the int8 kernel is what ran
    np.testing.assert_array_equal(got, oz.gemm_nt(A, B, C, alpha=-1.0, S=S))
