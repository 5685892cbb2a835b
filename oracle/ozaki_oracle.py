"""ozaki_oracle.py -- NumPy restatement of the int8 digit-plane GEMM of gpax_b200/csrc/ozaki.cuh.  TEST INFRASTRUCTURE ONLY.

The CUDA kernel evaluates  C += alpha * A B^T  (A [m,k], B [n,k], fp64) as S(S+1)/2 exact int8 x int8 -> int32 products
of digit planes plus a fixed-order fp64 recombination.  Every step of that is either exact integer arithmetic or a single
correctly rounded fp64 operation, so the whole computation can be restated on the CPU **bit for bit**:

  slice (oz_slice_kernel):   e_i = exponent of max_k |a_ik| (frexp), I = rint(a * 2^(8 S - 2 - e_i)) as a 64-bit integer
                             (one rounding, |I| <= 2^(8 S - 2)); its S base-256 digits in two's-complement style, lowest
                             first: d = signed low byte of I in [-128, 127], I = (I - d) >> 8; the top digit is what is
                             left (|d_0| <= 65).  a ~ 2^e_i * sum_q d_q 2^-(6 + 8 q)                -- exact integer steps
  products (oz_mma_kernel):  D_t = sum over digit pairs (p, q) with p + q = t of  A_p B_q^T        -- exact integers
  recombine (epilogue):      acc = 0; for t = S-1 .. 0: acc = fma(D_t, 2^-(12 + 8 t), acc)         -- D_t * 2^x is exact,
                                                                                                     one rounding per t
                             C = fma(2^e_i * alpha * 2^f_j, acc, C)                                -- exact product when
                                                                                                     alpha = +-1 (the only
                                                                                                     values the solver uses)
This module is the checker for that path (tests/test_ozaki_oracle.py pins its error bounds on the CPU; the GPU test
compares the kernel's output with it for equality).  Only tests/ may import it."""
import numpy as np


K_MAX = 16384      # int32 accumulation bound of one launch: S pairs per class * k * 2^14 < 2^31 for S <= 7


def slice_rows(A, S):
    """Digit planes [S, rows, k] (int64; plane 0 in [-65, 65], the others in [-128, 127]) and the row scales 2^e of
    oz_slice_kernel."""
    A = np.asarray(A, dtype=np.float64)
    mx = np.abs(A).max(axis=1) if A.shape[1] else np.zeros(A.shape[0])
    _, e = np.frexp(mx)                                   # mx = f * 2^e, f in [0.5, 1)
    e = np.where((mx > 0) & (mx < 1e300), e, 0).astype(np.int64)
    e = np.maximum(e, -900)                               # the kernel clamps too: 2^(8 S - 2 - e) must stay finite
    I = np.rint(np.ldexp(A, (8 * S - 2 - e)[:, None].astype(np.int32))).astype(np.int64)
    planes = np.empty((S,) + A.shape, dtype=np.int64)
    for q in range(S - 1, 0, -1):
        d = ((I + 128) & 0xff) - 128                      # signed low byte
        planes[q] = d
        I = (I - d) >> 8
    planes[0] = I
    return planes, np.ldexp(1.0, e.astype(np.int32))


def class_sums(PA, PB):
    """D_t = sum_{p+q=t} A_p B_q^T for t < S, as exact int64 (the int32 register accumulators hold the same values)."""
    S = PA.shape[0]
    D = np.zeros((S, PA.shape[1], PB.shape[1]), dtype=np.int64)
    FA, FB = PA.astype(np.float64), PB.astype(np.float64)     # |digit| <= 128, k <= 16384: every dot product is below 2^28,
    for p in range(S):                                        # so the float64 BLAS product is exact
        for q in range(S - p):
            D[p + q] += np.rint(FA[p] @ FB[q].T).astype(np.int64)
    return D


def gemm_nt(A, B, C, alpha=-1.0, S=7, lower_only=False):
    """C + alpha * A B^T exactly as the CUDA path rounds it.  alpha must be +-1 (power-of-two scale -> exact product).
    lower_only needs m >= n and follows the kernel's trapezoid rule (ozaki.cuh, OzMode): rows i < n update j <= i only, the
    rows below the square part update all n columns; every other entry is C unchanged."""
    if abs(alpha) != 1.0:
        raise ValueError("bit-exact restatement needs alpha = +-1")
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    if lower_only and A.shape[0] < B.shape[0]:
        raise ValueError("lower_only needs m >= n")
    if A.shape[1] > K_MAX:                                    # the library splits longer k into launches of <= K_MAX
        out = np.asarray(C, dtype=np.float64)
        for k0 in range(0, A.shape[1], K_MAX):
            out = gemm_nt(A[:, k0:k0 + K_MAX], B[:, k0:k0 + K_MAX], out, alpha, S, lower_only)
        return out
    PA, sa = slice_rows(A, S)
    PB, sb = slice_rows(B, S)
    D = class_sums(PA, PB)
    assert np.abs(D).max() < 2 ** 31, "int32 accumulator overflow"
    acc = np.zeros(D.shape[1:])
    for t in range(S - 1, -1, -1):
        acc = D[t].astype(np.float64) * np.ldexp(1.0, -(12 + 8 * t)) + acc      # exact product, one rounding: the fma
    out = (sa[:, None] * alpha * sb[None, :]) * acc + np.asarray(C, dtype=np.float64)
    if lower_only:
        out = np.where(np.tril(np.ones(out.shape, bool)), out, C)      # j <= i: for rows i >= n that is the whole row
    return out
