"""Operand rounding of the moment kernel's precisions at the bench's config-2 data (rcca workload: n = 100 000,
d = [1024, 1024], k = 64, c = 0.1), propagated to the rCCA weights.  Accumulation is exact (float64), so only the
operand formats differ:
    3xtf32 : hi*hi + hi*lo + lo*hi                      hi = trunc_tf32(x), lo = rna_tf32(x - hi)   (tf32x3)
    x3b    : hi*hi + bf16(hi)*bf16(x-hi) + bf16(x-hi)*bf16(hi)    bf16 = round to nearest even    (tf32x3b)
Prints the normalised covariance error and the max / median relative weight error per canonical vector against the
float64 covariance of the same float32 inputs (oracle.restatement.cov_rcca_fit on both).

    python tools/next/emulate_x3b_cfg2.py        # ~1 min and ~12 GB of host memory
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import restatement as R  # noqa: E402


def trunc_tf32(x):
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def rna_tf32(x):
    u = x.view(np.uint32).astype(np.uint64)
    return ((u + np.uint64(0x1000)) & np.uint64(0xFFFFE000)).astype(np.uint32).view(np.float32)


def rne_bf16(x):
    u = x.view(np.uint32).astype(np.uint64)
    u = (u + np.uint64(0x7FFF) + ((u >> np.uint64(16)) & np.uint64(1))) & np.uint64(0xFFFF0000)
    return u.astype(np.uint32).view(np.float32)


def covariance(M, s, n):
    return (M - np.outer(s, s) / n) / (n - 1)


def weight_errors(w, w_ref):
    w = R.align_signs(w, w_ref)
    return np.concatenate([np.linalg.norm(a - r, axis=0) / np.linalg.norm(r, axis=0) for a, r in zip(w, w_ref)])


def main():
    W = bench.W
    views = bench.make_views(1000)
    X = np.hstack(views).astype(np.float32)
    n, dims = X.shape[0], W["dims"]
    s = X.astype(np.float64).sum(axis=0)
    hi = trunc_tf32(X)
    lo = X - hi   # exact in float32
    hi64 = hi.astype(np.float64)
    HH = hi64.T @ hi64
    X64 = X.astype(np.float64)
    exact = covariance(X64.T @ X64, s, n)
    del X64
    lo3 = rna_tf32(lo).astype(np.float64)
    cross3 = hi64.T @ lo3
    bhi, blo = rne_bf16(hi).astype(np.float64), rne_bf16(lo).astype(np.float64)
    crossb = bhi.T @ blo
    del lo3, bhi, blo
    variants = {"3xtf32": covariance(HH + cross3 + cross3.T, s, n),
                "x3b": covariance(HH + crossb + crossb.T, s, n)}
    w_ref, _ = R.cov_rcca_fit(exact, dims, W["k"], W["c"], n)
    scale = np.sqrt(np.outer(np.diag(exact), np.diag(exact)))
    for name, C in variants.items():
        w, _ = R.cov_rcca_fit(C, dims, W["k"], W["c"], n)
        e = weight_errors(w, w_ref)
        print(f"{name:8s}: covariance {(np.abs(C - exact) / scale).max():.1e}  weights max {e.max():.1e}  "
              f"median {np.median(e):.1e}")


if __name__ == "__main__":
    main()
