"""TEST INFRASTRUCTURE — CPU oracle for the inverse-dynamics regressor (NumPy, fp64, batched).

Inverse dynamics ``u = M ddq + C dq - g`` is linear in the diagonal link inertias, so column p of the regressor
``Y(q, dq, ddq)`` is the inverse dynamics of the same chain with ``link_inertia = e_p``: parameter p = 6 (l - 1) + c is
``link_inertia[l][c]`` (l = 1..n, c = m_x, m_y, m_z, I_xx, I_yy, I_zz).  Each column is evaluated with
``rbd_oracle.ChainOracle``'s literal product-rule M, C and g, not with the joint-axis operators of the CUDA code
(abr_control_b200/csrc/abrb_regress.cuh), so the two are independent.
"""
import copy

import numpy as np

from . import rbd_oracle


def unit_chain(desc, p):
    """``desc`` with every link inertia zero except parameter p = 6 (l - 1) + c, which is 1"""
    d = copy.deepcopy(rbd_oracle.load_desc(desc) if isinstance(desc, str) else desc)
    W = np.zeros((d["n_links"], 6))
    W[1 + p // 6, p % 6] = 1.0
    d["link_inertia"] = W.tolist()
    return d


def inverse_dynamics(desc, q, dq, ddq):
    """(B, n): M ddq + C dq - g of the chain ``desc`` (an arm name or a descriptor dict)"""
    ch = rbd_oracle.ChainOracle(desc)
    q, dq, ddq = (np.atleast_2d(np.asarray(a, dtype=np.float64)) for a in (q, dq, ddq))
    return (np.einsum("bij,bj->bi", ch.M(q), ddq) + np.einsum("bij,bj->bi", ch.C(q, dq), dq) - ch.g(q))


def regressor(desc, q, dq, ddq):
    """(B, n, 6n): Y with ``Y @ theta == inverse_dynamics(desc, ...)``, theta = link_inertia[1:] flattened"""
    d = rbd_oracle.load_desc(desc) if isinstance(desc, str) else desc
    n = d["n_joints"]
    return np.stack([inverse_dynamics(unit_chain(d, p), q, dq, ddq) for p in range(6 * n)], axis=2)


def theta(desc):
    """(6n,) the inertial parameters of ``desc``"""
    d = rbd_oracle.load_desc(desc) if isinstance(desc, str) else desc
    return np.asarray(d["link_inertia"], dtype=np.float64)[1:].reshape(-1)
