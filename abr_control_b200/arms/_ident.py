"""Least-squares identification of the diagonal link inertias from recorded motion (``BaseConfig.identify_link_inertia``).

Inverse dynamics is linear in theta = link_inertia[1:] flattened, ``u = Y(q, dq, ddq) theta`` (include/abrb.h,
abrb_inverse_dynamics_regressor_*).  The three mass entries of a link are one unknown, so the fit runs on the tied
parameters phi = (m, I_xx, I_yy, I_zz) per link, ``theta = T phi`` and ``Y_r = Y T``.  The normal equations
``G = sum Y_r^T Y_r`` and ``c = sum Y_r^T (u - Y_r phi_0)`` are accumulated in fp64 over chunks of samples, so ``Y``
is never materialised for the whole record; the small symmetric solve runs on the host.
"""
import numpy as np
import torch

# columns whose norm is at or below this fraction of the largest are structurally zero (the regressor entry is a
# rounding residue of a product with an exactly zero axis component, ~1e-16 of the scale)
ZERO_COLUMN = 1e-12


def tie_matrix(n):
    """(6n, 4n): theta = T phi, phi = (m, I_xx, I_yy, I_zz) per link"""
    T = np.zeros((6 * n, 4 * n))
    for l in range(n):
        T[6 * l:6 * l + 3, 4 * l] = 1.0
        for c in range(3):
            T[6 * l + 3 + c, 4 * l + 1 + c] = 1.0
    return T


def tied(theta, n):
    """theta (6n,) -> phi (4n,); raises if a link's three mass entries differ"""
    W = np.asarray(theta, dtype=np.float64).reshape(n, 6)
    bad = [l + 1 for l in range(n) if not (W[l, 0] == W[l, 1] == W[l, 2])]
    if bad:
        raise ValueError(f"identify_link_inertia ties the mass entries of a link; link(s) {bad} of the prior model "
                         "have unequal m_x, m_y, m_z")
    return W[:, [0, 3, 4, 5]].reshape(-1)


def solve(G, c, rcond):
    """Least-squares solution of the normal equations ``G x = c`` with no component in the directions the data does
    not determine.  The rank decision is made on the equilibrated ``D^-1 G D^-1`` (D = sqrt(diag G)): its
    eigen-directions with eigenvalue ``<= rcond`` times the largest, and the structurally zero columns, are the null
    space.  ``x`` is then the minimum-norm solution in the coordinates of ``x`` (orthogonal to that null space), so a
    parameter is moved from the prior only as far as the data asks: the equilibrated coordinates would move a barely
    excited parameter arbitrarily far to absorb the null components of the others.

    -> (x, directions, zero): ``directions`` (len(c), rank), orthonormal, spans the row space of the regressor (the
    linear functionals of the parameters the data determines); ``zero`` marks the structurally zero columns."""
    m = len(c)
    d = np.sqrt(np.maximum(np.diag(G), 0.0))
    zero = d <= ZERO_COLUMN * d.max() if d.max() > 0 else np.ones(m, dtype=bool)
    live = ~zero
    x = np.zeros(m)
    null = [np.eye(m)[:, zero]]
    if live.any():
        dl = d[live]
        lam, V = np.linalg.eigh(G[np.ix_(live, live)] / np.outer(dl, dl))
        keep = lam > rcond * lam.max()
        x[live] = (V[:, keep] @ ((V[:, keep].T @ (c[live] / dl)) / lam[keep])) / dl
        Nd = np.zeros((m, int((~keep).sum())))
        Nd[live] = V[:, ~keep] / dl[:, None]  # null directions of the regressor in x coordinates
        null.append(Nd / np.linalg.norm(Nd, axis=0))
    N = np.hstack(null)
    Q = np.linalg.qr(N, mode="complete")[0] if N.shape[1] else np.eye(m)
    null_basis, directions = Q[:, :N.shape[1]], Q[:, N.shape[1]:]
    return x - null_basis @ (null_basis.T @ x), directions, zero


def identify(regress, K, chunk, theta0, rcond):
    """``regress(i0, i1)`` -> (Y (b, n, 6n), u (b, n)) torch tensors of samples i0 .. i1-1 (one device).  -> (theta,
    info) as ``BaseConfig.identify_link_inertia``."""
    n = theta0.size // 6
    phi0 = tied(theta0, n)
    T = tie_matrix(n)
    G = c = None
    ss = [0.0, 0.0]

    def reduced(i0, i1):
        Y, u = regress(i0, i1)
        Tt = torch.as_tensor(T, device=Y.device)
        return torch.matmul(Y.to(torch.float64), Tt).reshape(-1, 4 * n), u.to(torch.float64).reshape(-1)

    p0 = None
    for i0 in range(0, K, chunk):
        Yr, u = reduced(i0, min(K, i0 + chunk))
        if G is None:
            G = torch.zeros((4 * n, 4 * n), dtype=torch.float64, device=Yr.device)
            c = torch.zeros(4 * n, dtype=torch.float64, device=Yr.device)
            p0 = torch.as_tensor(phi0, device=Yr.device)
        r = u - torch.matmul(Yr, p0)
        G += torch.matmul(Yr.T, Yr)
        c += torch.matmul(Yr.T, r)
        ss[0] += float(torch.dot(r, r))
    dphi, directions, zero = solve(G.cpu().numpy(), c.cpu().numpy(), rcond)
    phi = phi0 + dphi
    p1 = torch.as_tensor(phi, device=G.device)
    for i0 in range(0, K, chunk):
        Yr, u = reduced(i0, min(K, i0 + chunk))
        r = u - torch.matmul(Yr, p1)
        ss[1] += float(torch.dot(r, r))
    # a functional w . phi is the functional (T (T^T T)^-1 w) . theta on tied theta
    basis = np.linalg.qr(T @ (directions / np.diag(T.T @ T)[:, None]))[0]
    unident = [int(p) for j in np.flatnonzero(zero) for p in np.flatnonzero(T[:, j])]
    info = dict(rank=int(directions.shape[1]), basis=basis, unidentifiable=unident,
                rms_before=float(np.sqrt(ss[0] / (K * n))), rms_after=float(np.sqrt(ss[1] / (K * n))))
    return T @ phi, info
