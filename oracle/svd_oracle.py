"""TEST INFRASTRUCTURE ONLY -- the spectral-norm penalty (bm/svd.py over torch.svd_lowrank) restated in fp64 with the draws
injected, value and gradient, as brainmagick_b200.svd computes them (DESIGN §4.10):

  A = the weight viewed as [shape[0], -1], transposed when it is wide (m < n, as torch.svd_lowrank does), R [n, q];
  n <= q:  the span is A's whole range: λ = σ₁(A)², dλ/dA = 2 σ₁ u₁ v₁ᵀ;
  else:    Q = orth(A R), then niter times Q = orth(Aᵀ Q), Q = orth(A Q);  λ = λmax(Qᵀ A Aᵀ Q) with eigenvector w, and the
           gradient through the spans: z = Q w, dA = 2 z zᵀ A, gQ = 2 (A Aᵀ z) wᵀ, then for every step X = Y Rx in reverse
           gX = (I - Y Yᵀ) gQ Rx⁻ᵀ; X = A Qin adds gX Qinᵀ and passes gQin = Aᵀ gX, X = Aᵀ Qin adds Qin gXᵀ and passes A gX.

The orthonormalisation is torch.linalg.qr: only the span enters, so any orthonormal basis gives the same λ and gradient.
"""
from __future__ import annotations

import typing as tp

import torch


def estimate(p2d: torch.Tensor, R: torch.Tensor, niter: int = 2) -> tp.Tuple[float, torch.Tensor]:
    """(λ, dλ/dp2d) in fp64 for one weight p2d [rows, cols] and its draw R [min(rows, cols), q]"""
    P = p2d.detach().double()
    wide = P.shape[0] < P.shape[1]
    A = P.T if wide else P
    R = R.double()
    n, q = A.shape[1], R.shape[1]
    if n <= q:
        lam, V = torch.linalg.eigh(A.T @ A)
        v = V[:, -1]
        s2, gA = lam[-1], 2 * torch.outer(A @ v, v)
    else:
        steps = []                               # (Y, Rx, kind, Qin): X = Y Rx, X = A Qin ("A") or Aᵀ Qin ("At")
        Q, Rx = torch.linalg.qr(A @ R)
        steps.append((Q, Rx, "A", R))
        for _ in range(niter):
            Qin = Q
            Q, Rx = torch.linalg.qr(A.T @ Qin)
            steps.append((Q, Rx, "At", Qin))
            Qin = Q
            Q, Rx = torch.linalg.qr(A @ Qin)
            steps.append((Q, Rx, "A", Qin))
        Yt = A.T @ Q
        lam, W = torch.linalg.eigh(Yt.T @ Yt)
        w, s2 = W[:, -1], lam[-1]
        z = Q @ w
        gA = 2 * torch.outer(z, A.T @ z)
        gQ = 2 * torch.outer(A @ (A.T @ z), w)
        for Y, Rx, kind, Qin in reversed(steps):
            gX = torch.linalg.solve_triangular(Rx, (gQ - Y @ (Y.T @ gQ)).T, upper=True, left=True).T   # (...) Rx⁻ᵀ
            if kind == "A":
                gA = gA + gX @ Qin.T
                gQ = A.T @ gX
            else:
                gA = gA + Qin @ gX.T
                gQ = A @ gX
    return float(s2), (gA.T if wide else gA)


def penalty(weights: tp.Sequence[torch.Tensor], draws: tp.Sequence[torch.Tensor], niter: int = 2,
            proba: float = 1.0) -> tp.Tuple[float, tp.List[torch.Tensor]]:
    """(Σ λ / proba, [dvalue/dweight in each weight's own shape]) in fp64"""
    total, grads = 0.0, []
    for p, R in zip(weights, draws):
        s2, g = estimate(p.reshape(p.shape[0], -1), R, niter)
        total += s2
        grads.append((g / proba).reshape(p.shape))
    return total / proba, grads


def reference_algorithm(p2d: torch.Tensor, R: torch.Tensor, niter: int = 2) -> torch.Tensor:
    """torch.svd_lowrank(p2d, q, niter)[1][0] ** 2 with the draw R injected, in p2d's dtype and differentiable through
    torch's QR and SVD -- what bm/svd.py computes, used to measure the reference's own rounding error"""
    A = p2d.mT if p2d.shape[0] < p2d.shape[1] else p2d
    Q = torch.linalg.qr(A @ R).Q
    for _ in range(niter):
        Q = torch.linalg.qr(A.mT @ Q).Q
        Q = torch.linalg.qr(A @ Q).Q
    return torch.linalg.svd(Q.mT @ A, full_matrices=False)[1][0] ** 2
