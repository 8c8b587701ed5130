"""Batched ``robot_config``: the reference's arm-model duck type, evaluated on the GPU.

Mirrors the public methods of ``abr_control.arms.base_config.BaseConfig``
(/root/reference/abr_control/arms/base_config.py:210-415) — same names, same argument order:

    g(q)  dJ(name, q, dq, x=None)  J(name, q, x=None)  M(q)  R(name, q)  quaternion(name, q)
    C(q, dq)  T(name, q)  Tx(name, q, x=None)  T_inv(name, q, x=None)

Each accepts
  * ONE state — ``q`` of shape ``(n,)`` (list / NumPy): returns exactly the reference's shapes and dtypes
    (``J, dJ, M, g, C, R`` rounded to float32 as base_config.py:223,247,270,285,301,336 do; ``Tx, T, T_inv``
    float64), as fresh writable ndarrays;
  * a BATCH — ``q`` of shape ``(B, n)``: NumPy in -> NumPy out (host buffers, copies inside the call), or a CUDA
    ``torch.Tensor`` in -> CUDA tensors out on the current torch stream (no host round trip).  Batched results
    keep the compute dtype (float64 by default, float32 for float32 inputs) and are stacked along axis 0.

All arithmetic runs in hand-written sm_90a kernels behind ``libabrb.so``; there is no SymPy, no code
generation, no cache directory and no CPU fallback.
"""
import ctypes as C

import numpy as np

from .. import _abi, _lib
from ..controllers._batch import host_out as _host_out

try:  # torch is only needed when the caller hands in CUDA tensors
    import torch
except Exception:  # pragma: no cover
    torch = None

_RBD_KEYS = ("Tx", "T", "R", "T_inv", "quat", "J", "dJ", "M", "g", "C")


def _is_torch(x):
    return torch is not None and isinstance(x, torch.Tensor)


def _is_torch_grad(*xs):
    """grad mode is on and one of ``xs`` is a tensor that requires grad (the differentiable path of the plant)"""
    return torch.is_grad_enabled() and any(_is_torch(x) and x.requires_grad for x in xs)


class BaseConfig:
    """Batched arm model built from a flat chain descriptor (see ``abr_control_b200/arms/data/*.json``).

    Parameters
    ----------
    desc : dict
        chain descriptor: n_joints, n_links, L0, A, B, E (3x4 blocks), link_inertia, gravity
    dtype : numpy dtype, optional (Default: float64)
        compute precision used for host (NumPy / list) inputs; CUDA tensors use their own dtype
    """

    def __init__(self, desc, ROBOT_NAME="robot", dtype=np.float64, **kwargs):
        kwargs.pop("use_cython", None)  # accepted for signature compatibility (base_config.py:78); meaningless here
        if kwargs:
            raise TypeError(f"unexpected arguments {sorted(kwargs)}")
        self.desc = desc
        self.ROBOT_NAME = ROBOT_NAME
        self.N_JOINTS = int(desc["n_joints"])
        self.N_LINKS = int(desc["n_links"])
        self.dtype = np.dtype(dtype)
        if self.dtype not in (np.dtype(np.float32), np.dtype(np.float64)):
            raise ValueError("dtype must be float32 or float64")
        self._cdesc = _abi.chain_desc_from_dict(desc)
        self._M_LINKS = [np.diag(row) for row in np.asarray(desc["link_inertia"], dtype=float)]
        self._M_JOINTS = [np.zeros((6, 6)) for _ in range(self.N_JOINTS)]
        self.L = np.asarray(desc.get("L", []), dtype=float)
        self.START_ANGLES = np.asarray(desc.get("start_angles", np.zeros(self.N_JOINTS)), dtype=float)
        self.x_zeros = np.zeros(3)
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().abrb_model_create(C.byref(self._cdesc), C.byref(self._handle)))
        self._frame_ids = {}

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                _lib.lib().abrb_model_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    # ------------------------------------------------------------------ helpers
    @property
    def handle(self):
        return self._handle

    @property
    def is_orthonormal(self):
        return bool(_lib.lib().abrb_model_is_orthonormal(self._handle))

    def frame_id(self, name):
        """Frame name -> id.  Unknown names raise like the reference (arms/ur5/config.py:336-337)."""
        fid = self._frame_ids.get(name)
        if fid is None:
            fid = _lib.lib().abrb_frame_id(self._handle, str(name).encode())
            if fid < 0:
                raise Exception(f"Invalid transformation name: {name}")
            self._frame_ids[name] = fid
        return fid

    def _shapes(self):
        n = self.N_JOINTS
        return dict(Tx=(3,), T=(4, 4), R=(3, 3), T_inv=(4, 4), quat=(4,), J=(6, n), dJ=(6, n), M=(n, n), g=(n,),
                    C=(n, n))

    def _prep(self, arr, dtype=None):
        """-> (array as (B,n) contiguous, single?, kind) where kind is 'torch' or 'numpy'."""
        n = self.N_JOINTS
        if _is_torch(arr):
            if not arr.is_cuda:
                raise ValueError("torch inputs must be CUDA tensors (use NumPy for host data)")
            if arr.dtype not in (torch.float32, torch.float64):
                raise ValueError("torch inputs must be float32 or float64")
            single = arr.dim() == 1
            a = arr.reshape(1, -1) if single else arr
            if a.dim() != 2 or a.shape[1] != n:
                raise ValueError(f"expected shape ({n},) or (B, {n}), got {tuple(arr.shape)}")
            return a.contiguous(), single, "torch"
        a = np.asarray(arr, dtype=self.dtype if dtype is None else dtype)
        single = a.ndim == 1
        a = a.reshape(1, -1) if single else a
        if a.ndim != 2 or a.shape[1] != n:
            raise ValueError(f"expected shape ({n},) or (B, {n}), got {np.shape(arr)}")
        return np.ascontiguousarray(a), single, "numpy"

    def eval(self, q, dq=None, name="EE", x=None, want=("J", "M", "g")):
        """Evaluate several quantities in ONE kernel launch.  Returns a dict keyed like ``want``.

        This is the batched superset of the reference's one-quantity-per-call methods; the individual
        methods below call it with a single key.
        """
        want = tuple(want)
        for k in want:
            if k not in _RBD_KEYS:
                raise KeyError(k)
        qa, single, kind = self._prep(q, np.float64 if np.ndim(q) == 1 and not _is_torch(q) else None)
        need_dq = ("dJ" in want) or ("C" in want)
        dqa = None
        if dq is not None:
            dqa, _, kind2 = self._prep(dq, qa.dtype if kind == "numpy" else None)
            if kind2 != kind or dqa.shape != qa.shape or (kind == "torch" and dqa.dtype != qa.dtype):
                raise ValueError("q and dq must have the same type, dtype and shape")
        elif need_dq:
            raise ValueError("dq is required for dJ / C")
        fid = self.frame_id(name)
        xo = None
        if x is not None and not np.allclose(np.asarray(x, dtype=float), 0):
            xo = (C.c_double * 3)(*[float(v) for v in np.asarray(x, dtype=float).reshape(3)])
        B = qa.shape[0]
        shapes = self._shapes()
        out = _abi.RbdOut()
        res = {}
        L = _lib.lib()
        if kind == "torch":
            f32 = qa.dtype == torch.float32
            with torch.cuda.device(qa.device):
                for k in want:
                    res[k] = torch.empty((B,) + shapes[k], dtype=qa.dtype, device=qa.device)
                    setattr(out, k, res[k].data_ptr())
                fn = L.abrb_rbd_eval_f32 if f32 else L.abrb_rbd_eval_f64
                stream = torch.cuda.current_stream(qa.device).cuda_stream
                _lib.check(fn(self._handle, fid, xo, qa.data_ptr(), dqa.data_ptr() if dqa is not None else None, B,
                              C.byref(out), stream))
        else:
            f32 = qa.dtype == np.float32
            for k in want:
                res[k] = _host_out((B,) + shapes[k], qa.dtype)
                setattr(out, k, res[k].ctypes.data)
            fn = L.abrb_rbd_eval_host_f32 if f32 else L.abrb_rbd_eval_host_f64
            _lib.check(fn(self._handle, fid, xo, qa.ctypes.data, dqa.ctypes.data if dqa is not None else None, B,
                          C.byref(out)))
        if single:
            res = {k: v[0] for k, v in res.items()}
        return res

    def eval_into(self, q, dq, out, name="EE", x=None):
        """Allocation-free batched evaluation for hot loops: ``q``/``dq`` contiguous CUDA tensors (B, n) of one dtype,
        ``out`` a dict key -> preallocated contiguous CUDA tensor of the right shape (keys as in ``eval``)."""
        B = q.shape[0]
        if not q.is_cuda or q.dim() != 2 or q.shape[1] != self.N_JOINTS or not q.is_contiguous():
            raise ValueError("eval_into: q must be a contiguous CUDA tensor of shape (B, n_joints)")
        if dq is not None and (dq.shape != q.shape or dq.dtype != q.dtype or dq.device != q.device or not dq.is_contiguous()):
            raise ValueError("eval_into: dq must match q")
        o = _abi.RbdOut()
        shapes = self._shapes()
        for k, t in out.items():
            if k not in _RBD_KEYS or t.dtype != q.dtype or not t.is_contiguous() or t.device != q.device:
                raise ValueError(f"eval_into: bad output {k}")
            if tuple(t.shape) != (B,) + shapes[k]:
                raise ValueError(f"eval_into: output {k} must have shape {(B,) + shapes[k]}")
            setattr(o, k, t.data_ptr())
        xo = None
        if x is not None:
            xo = (C.c_double * 3)(*[float(v) for v in x])
        L = _lib.lib()
        fn = L.abrb_rbd_eval_f32 if q.dtype == torch.float32 else L.abrb_rbd_eval_f64
        with torch.cuda.device(q.device):  # the launch goes to the tensors' device, whatever the current one is
            _lib.check(fn(self._handle, self.frame_id(name), xo, q.data_ptr(), None if dq is None else dq.data_ptr(), B,
                          C.byref(o), torch.cuda.current_stream(q.device).cuda_stream))
        return out

    def _one(self, key, q, dq=None, name="EE", x=None, ref32=False):
        v = self.eval(q, dq=dq, name=name, x=x, want=(key,))[key]
        if isinstance(v, np.ndarray) and v.ndim == len(self._shapes()[key]):
            # single state: the reference's dtype contract
            return np.array(v, dtype="float32") if ref32 else np.array(v, dtype=np.float64)
        return v

    # ------------------------------------------------------------------ the reference's public surface
    def g(self, q):
        """Joint-space gravity force (base_config.py:210-223)."""
        return self._one("g", q, ref32=True)

    def dJ(self, name, q, dq, x=None):
        """Time derivative of the Jacobian (base_config.py:225-247)."""
        return self._one("dJ", q, dq=dq, name=name, x=x, ref32=True)

    def J(self, name, q, x=None):
        """6 x n Jacobian of point ``x`` in frame ``name`` (base_config.py:249-270)."""
        return self._one("J", q, name=name, x=x, ref32=True)

    def M(self, q):
        """Joint-space inertia matrix (base_config.py:272-285)."""
        return self._one("M", q, ref32=True)

    def R(self, name, q):
        """Rotation matrix of frame ``name`` (base_config.py:287-301)."""
        return self._one("R", q, name=name, ref32=True)

    def quaternion(self, name, q):
        """Unit quaternion (w, x, y, z) of frame ``name`` (base_config.py:304-318)."""
        return self._one("quat", q, name=name)

    def C(self, q, dq):
        """Centrifugal/Coriolis matrix such that ``C @ dq`` is the force (base_config.py:320-336)."""
        return self._one("C", q, dq=dq, ref32=True)

    def T(self, name, q):
        """4 x 4 transform of frame ``name`` (base_config.py:338-369)."""
        return self._one("T", q, name=name)

    def Tx(self, name, q, x=None):
        """World position of point ``x`` of frame ``name`` (base_config.py:371-392)."""
        return self._one("Tx", q, name=name, x=x)

    def T_inv(self, name, q, x=None):
        """Inverse transform [[R^T, -R^T t], [0, 1]] (base_config.py:394-415; ``x`` is unused there too)."""
        return self._one("T_inv", q, name=name)

    # ------------------------------------------------------------------ the plant (include/abrb.h, abrb_plant_*)
    def _on_device(self, q, dq):
        """-> (q, dq as CUDA tensors (B, n), single?, 'torch' or 'numpy', f32?); NumPy is staged through the current
        device."""
        from ..controllers import _batch

        qa, dqa, single, kind, f32 = _batch.prep_state(self, q, dq)
        if kind == "numpy":
            dev = torch.device("cuda", torch.cuda.current_device())
            qa, dqa = torch.as_tensor(qa).to(dev), torch.as_tensor(dqa).to(dev)
        return qa, dqa, single, kind, f32

    def _on_device_rows(self, q, dq, x, what):
        """``_on_device`` and a third ``(B, n)`` input ``x`` of the same form -> (q, dq, x, single, kind, f32)"""
        qa, dqa, single, kind, f32 = self._on_device(q, dq)
        B, n = qa.shape
        xa = (x if _is_torch(x) else torch.as_tensor(np.asarray(x, dtype=np.float64))).to(device=qa.device,
                                                                                            dtype=qa.dtype)
        if tuple(xa.shape) != ((n,) if single else (B, n)):
            raise ValueError(f"{what} must have the shape of q, ({n},) or ({B}, {n}), got {tuple(xa.shape)}")
        return qa, dqa, xa.reshape(B, n).contiguous(), single, kind, f32

    def _dynamics(self, q, dq, x, what, fns):
        qa, dqa, xa, single, kind, f32 = self._on_device_rows(q, dq, x, what)
        B = qa.shape[0]
        out = torch.empty_like(qa)
        fn = getattr(_lib.lib(), fns[1] if f32 else fns[0])
        with torch.cuda.device(qa.device):
            _lib.check(fn(self._handle, qa.data_ptr(), dqa.data_ptr(), xa.data_ptr(), out.data_ptr(), B,
                          torch.cuda.current_stream(qa.device).cuda_stream))
        if kind == "numpy":
            out = out.cpu().numpy()
        return out[0] if single else out

    def _derivatives(self, q, dq, x, kind, want_in=True):
        qa, dqa, xa, single, hkind, f32 = self._on_device_rows(q, dq, x, "u" if kind == 0 else "ddq")
        B, n = qa.shape
        d = [torch.empty((B, n, n), dtype=qa.dtype, device=qa.device) for _ in range(3 if want_in else 2)]
        name = "abrb_forward_dynamics_derivatives" if kind == 0 else "abrb_inverse_dynamics_derivatives"
        fn = getattr(_lib.lib(), name + ("_f32" if f32 else "_f64"))
        with torch.cuda.device(qa.device):
            _lib.check(fn(self._handle, qa.data_ptr(), dqa.data_ptr(), xa.data_ptr(), d[0].data_ptr(), d[1].data_ptr(),
                          d[2].data_ptr() if want_in else None, B, torch.cuda.current_stream(qa.device).cuda_stream))
        if hkind == "numpy":
            d = [t.cpu().numpy() for t in d]
        if single:
            d = [t[0] for t in d]
        return tuple(d) if want_in else (d[0], d[1], None)

    def _with_theta(self, theta):
        """The model with ``link_inertia[1:] = theta`` (``(6n,)``: a NumPy array or a float32/float64 CUDA tensor, read
        back to the host once: a device synchronisation), for the ``theta`` argument of the plant's methods."""
        if _is_torch(theta) and (not theta.is_cuda or theta.dtype not in (torch.float32, torch.float64)):
            raise ValueError("theta must be a NumPy array or a float32/float64 CUDA tensor")
        return self.with_link_inertia(theta)

    def forward_dynamics(self, q, dq, u, theta=None):
        """Joint accelerations under the torque ``u``: ``ddq = M(q)^-1 (u + g(q) - C(q, dq) dq)``, the plant of the
        rollouts (``g`` is the gravity force the controllers subtract, so ``u = -g`` holds the arm still).
        ``q, dq, u`` are ``(n,)`` or ``(B, n)``; CUDA tensors in -> CUDA tensors out, NumPy in -> NumPy out.
        Differentiable (``torch.autograd``, first order) when grad mode is on and a CUDA tensor input requires grad.

        ``theta`` (``(6n,)``, see ``inertial_parameters``): evaluate with ``link_inertia[1:] = theta``, exactly as
        ``with_link_inertia(theta).forward_dynamics(q, dq, u)`` (a tensor ``theta`` is read back to the host once per
        call to build that model, a device synchronisation).  A CUDA ``theta`` that requires grad is differentiable
        too: at fixed ``u``, ``Y(q, dq, ddq) theta = u`` gives ``d ddq / d theta = -M^-1 Y(q, dq, ddq)``, so
        ``theta.grad = -sum_b Y(q_b, dq_b, ddq_b)^T M_b^-1 g_b`` for the output cotangent ``g`` (``Y``:
        ``inverse_dynamics_regressor``)."""
        rc = self if theta is None else self._with_theta(theta)
        if torch is not None and _is_torch_grad(q, dq, u, theta):
            from . import _autograd

            return _autograd.dynamics(rc, 0, q, dq, u, theta)
        return rc._dynamics(q, dq, u, "u", ("abrb_forward_dynamics_f64", "abrb_forward_dynamics_f32"))

    def inverse_dynamics(self, q, dq, ddq, theta=None):
        """Torque that produces ``ddq``: ``u = M(q) ddq + C(q, dq) dq - g(q)`` (the inverse of ``forward_dynamics``),
        e.g. the feedforward torque of a planned joint trajectory.  Shapes and types as ``forward_dynamics``; likewise
        differentiable.  ``theta`` as in ``forward_dynamics``; ``u = Y(q, dq, ddq) theta`` is linear in it, so
        ``theta.grad = sum_b Y(q_b, dq_b, ddq_b)^T g_b``."""
        rc = self if theta is None else self._with_theta(theta)
        if torch is not None and _is_torch_grad(q, dq, ddq, theta):
            from . import _autograd

            return _autograd.dynamics(rc, 1, q, dq, ddq, theta)
        return rc._dynamics(q, dq, ddq, "ddq", ("abrb_inverse_dynamics_f64", "abrb_inverse_dynamics_f32"))

    # ------------------------------------------------------------------ inertial parameters
    def inverse_dynamics_regressor(self, q, dq, ddq):
        """Regressor ``Y`` of ``inverse_dynamics``, linear in the inertial parameters: ``Y @ inertial_parameters() ==
        inverse_dynamics(q, dq, ddq)`` (to rounding), column ``p = 6 (l - 1) + c`` being the torque per unit
        ``link_inertia[l][c]`` (links 1..n; c = m_x, m_y, m_z, I_xx, I_yy, I_zz).  ``(B, n, 6n)``, or ``(n, 6n)`` for
        one state: a view of the ``(B, 6n, n)`` record of ``abrb_inverse_dynamics_regressor_*``.  Input forms as
        ``inverse_dynamics`` (CUDA tensors in -> CUDA tensors out, NumPy in -> NumPy out, dtype of the input)."""
        qa, dqa, aa, single, kind, f32 = self._on_device_rows(q, dq, ddq, "ddq")
        B, n = qa.shape
        Yt = torch.empty((B, 6 * n, n), dtype=qa.dtype, device=qa.device)
        L = _lib.lib()
        fn = L.abrb_inverse_dynamics_regressor_f32 if f32 else L.abrb_inverse_dynamics_regressor_f64
        with torch.cuda.device(qa.device):
            _lib.check(fn(self._handle, qa.data_ptr(), dqa.data_ptr(), aa.data_ptr(), Yt.data_ptr(), B,
                          torch.cuda.current_stream(qa.device).cuda_stream))
        Y = Yt.cpu().numpy().transpose(0, 2, 1) if kind == "numpy" else Yt.transpose(1, 2)
        return Y[0] if single else Y

    def inertial_parameters(self):
        """``(6n,)`` float64: this model's ``link_inertia[1:]`` flattened, the ``theta`` of
        ``inverse_dynamics_regressor`` (link 0 never moves, so it never enters the dynamics)."""
        return np.asarray(self.desc["link_inertia"], dtype=np.float64)[1:].reshape(-1).copy()

    def with_link_inertia(self, theta):
        """A new model with the same chain, link 0 and precision, and ``link_inertia[1:] = theta`` (``(6n,)``, as
        ``inertial_parameters``)."""
        n = self.N_JOINTS
        th = np.asarray(theta.detach().cpu() if _is_torch(theta) else theta, dtype=np.float64)
        if th.shape != (6 * n,) or not np.all(np.isfinite(th)):
            raise ValueError(f"theta must be {6 * n} finite values, got shape {th.shape}")
        W = np.asarray(self.desc["link_inertia"], dtype=np.float64).copy()
        W[1:] = th.reshape(n, 6)
        return BaseConfig(dict(self.desc, link_inertia=W.tolist()), ROBOT_NAME=self.ROBOT_NAME, dtype=self.dtype)

    def identify_link_inertia(self, q, dq, ddq, u, rcond=1e-10, chunk_states=65536):
        """Least-squares fit of the link inertias to recorded motion: the ``theta`` that minimises ``|Y theta - u|``
        over the samples, starting from this model.  ``q, dq, ddq, u``: ``(K, n)`` samples (CUDA tensors, or NumPy
        staged through the current device in chunks).  Returns ``(theta, info)``; ``with_link_inertia(theta)`` is the
        identified model.

        * The three mass entries of a link are one unknown (this model's must be equal), so there are 4 per link.
        * ``G = sum Y^T Y`` and ``Y^T`` times the prior's residual are accumulated in fp64 over ``chunk_states``
          samples at a time with the device regressor (fp32 inputs give an fp32 regressor, accumulated in fp64).
        * Columns are equilibrated; structurally zero columns are dropped, as are eigen-directions of the equilibrated
          Gram matrix with eigenvalue ``<= rcond * largest``.  ``theta`` is the minimum-norm update of this model's
          parameters within the kept directions: what the data cannot see stays at the prior.
        * ``info``: ``rank`` (kept directions), ``basis`` (``(6n, rank)``, orthonormal: the identifiable directions in
          ``theta`` coordinates; compare models by their projections on it, not entry by entry),
          ``unidentifiable`` (indices of ``theta`` whose column is zero), ``rms_before`` / ``rms_after`` (RMS torque
          residual of this model and of the fit over all ``K n`` torques).

        Samples from a recorded rollout (``simulate``, or a controller's ``rollout_path``) from ``(q0, dq0)`` with step
        ``dt``: ``traj["u"][t]`` belongs to the state BEFORE step t and ``traj["q"][t]``, ``traj["dq"][t]`` to the state
        after it, so with ``q_prev = [q0, traj["q"][:-1]]`` and ``dq_prev`` likewise, the samples are ::

            q, dq = q_prev, dq_prev;  ddq = (traj["dq"] - dq_prev) / dt;  u = traj["u"]     # each (S, B, n)
            theta, info = rc.identify_link_inertia(*(a.reshape(-1, n) for a in (q, dq, ddq, u)))

        ``ddq`` is exact there (to rounding): the semi-implicit Euler step sets ``dq_{t+1} = dq_t + ddq_t dt``."""
        from . import _ident

        n = self.N_JOINTS
        theta0 = self.inertial_parameters()
        _ident.tied(theta0, n)
        if chunk_states < 1:
            raise ValueError("chunk_states must be >= 1")
        xs = [q, dq, ddq, u]
        on_device = all(_is_torch(x) for x in xs)
        if on_device:
            if not xs[0].is_cuda or any(x.device != xs[0].device or x.dtype != xs[0].dtype for x in xs):
                raise ValueError("q, dq, ddq and u must be CUDA tensors of one device and dtype, or NumPy arrays")
        elif any(_is_torch(x) for x in xs):
            raise ValueError("q, dq, ddq and u must be CUDA tensors of one device and dtype, or NumPy arrays")
        else:
            xs = [np.asarray(x, dtype=self.dtype) for x in xs]
        K = xs[0].shape[0] if xs[0].ndim == 2 else -1
        if K < 1 or any(tuple(x.shape) != (K, n) for x in xs):
            raise ValueError(f"q, dq, ddq and u must be (K, {n}) with K >= 1")
        if on_device:
            dev, dtype = xs[0].device, xs[0].dtype
        else:
            dev = torch.device("cuda", torch.cuda.current_device())
            dtype = torch.float32 if self.dtype == np.float32 else torch.float64

        def regress(i0, i1):
            qc, dqc, ac, uc = (torch.as_tensor(x[i0:i1]).to(device=dev, dtype=dtype) for x in xs)
            return self.inverse_dynamics_regressor(qc, dqc, ac), uc

        return _ident.identify(regress, K, int(chunk_states), theta0, float(rcond))

    def forward_dynamics_derivatives(self, q, dq, u):
        """Derivatives of ``forward_dynamics``: ``(d_q, d_dq, d_u)``, each ``(B, n, n)`` (``(n, n)`` for one state) with
        element ``[b, i, j] = d ddq_i / d x_j``; ``d_u`` is ``M^-1``.  Exact (forward-mode dual numbers through the
        same device code), not finite differences.  Input and output types as ``forward_dynamics``."""
        return self._derivatives(q, dq, u, 0)

    def inverse_dynamics_derivatives(self, q, dq, ddq):
        """Derivatives of ``inverse_dynamics``: ``(d_q, d_dq, d_ddq)``, element ``[b, i, j] = d u_i / d x_j``;
        ``d_ddq`` is ``M``.  Types and shapes as ``forward_dynamics_derivatives``."""
        return self._derivatives(q, dq, ddq, 1)

    def simulate(self, q, dq, u, dt=1e-3, path=None, effort_weight=0.0, compensate_gravity=False, ref_frame="EE",
                 xyz_offset=None, record=("q", "dq", "u", "x"), theta=None):
        """Open-loop rollout of the plant under the torque sequence ``u`` on the GPU (abrb_plant_rollout_*).  For each
        step ``t = 0 .. S-1``, with the semi-implicit Euler step of the reference (arms/twojoint/arm_sim.py:131-132)::

            tau_t = u[t]                    (or u[t] - g(q_t) with compensate_gravity: the residual-torque form)
            x_t   = Tx(ref_frame, q_t, x=xyz_offset)
            ddq   = M^-1 (tau_t + g - C dq_t);  dq_{t+1} = dq_t + ddq dt;  q_{t+1} = q_t + dq_{t+1} dt
            cost += |x_t - path[t, :3]|^2 (with a path) + effort_weight * |tau_t|^2

        ``u`` is ``(S, n)`` (one sequence for every trajectory) or ``(S, B, n)``; ``path`` is None, ``(S, 6)`` or
        ``(S, B, 6)`` as in ``OSC.rollout_path`` (only columns 0-2 are used).  Returns ``(q_final, dq_final, traj,
        cost)`` with the records of ``OSC.rollout_path``: ``traj[k]`` for k in ``record`` is ``(S, B, n)`` (``"x"``:
        ``(S, B, 3)``); ``traj["x"][t]`` and ``traj["u"][t]`` (the applied ``tau_t``) belong to the state before step
        t, ``traj["q"][t]`` and ``traj["dq"][t]`` to the state after it; ``cost`` is ``(B,)``.  ``record=()`` is the
        allocation-light form for sampling-based MPC, e.g. MPPI around a nominal torque plan::

            _, _, _, cost = rc.simulate(q0, dq0, u_nominal + noise, path=P, record=())    # noise (S, B, n)

        Fed the ``traj["u"]`` that ``OSC.rollout_path`` recorded, with the same start, path and effort weight, it gives
        back that rollout's track and cost, so closed-loop and open-loop candidates are scored alike::

            qf, dqf, tr, c = osc.rollout_path(q0, dq0, P, effort_weight=w)
            qs, dqs, ts, cs = rc.simulate(q0, dq0, tr["u"], path=P, effort_weight=w)       # ts["x"] == tr["x"]

        CUDA tensors in -> CUDA tensors out; NumPy in -> NumPy out.  A single state ``q`` of shape ``(n,)`` takes an
        ``(S, n)`` sequence and returns ``(S, n)`` records and a scalar cost.

        Differentiable (``torch.autograd``, first order) when grad mode is on and ``q``, ``dq`` or ``u`` is a CUDA
        tensor that requires grad: gradients reach ``u`` (summed over trajectories for a shared ``(S, n)`` sequence),
        ``q`` and ``dq`` from the cost, the final state and every returned record, through the adjoint recursion of
        ``abrb_plant_rollout_vjp_*``.  The path, ``dt`` and ``effort_weight`` are constants; a path that requires
        grad raises ``NotImplementedError``.

        ``theta`` (``(6n,)``, see ``inertial_parameters``): roll out the plant with ``link_inertia[1:] = theta``; values
        and records are those of ``with_link_inertia(theta).simulate(...)`` (a tensor ``theta`` is read back to the
        host once per call to build that model, a device synchronisation).  A CUDA ``theta`` that requires grad gets
        its gradient too (DESIGN.md S3.8, ``abrb_plant_rollout_theta_vjp_*`` after the adjoint recursion): with
        ``(q_t, dq_t)`` the state before step t, ``tau_t`` its applied torque, ``ddq_t = M^-1 (tau_t + g - C dq_t)``,
        ``gu_t`` the per-trajectory torque cotangent, ``gc_b`` the cost cotangent and ``gr_t`` that of
        ``traj["u"][t]``::

            w_t        = gu_t - 2 effort_weight gc_b tau_t - gr_t         (the part of gu_t that flows through ddq_t)
            theta.grad = sum_b sum_t [ -Y(q_t, dq_t, ddq_t)^T w_t + c_g Y(q_t, 0, 0)^T gu_t ]

        with ``c_g = 1`` under ``compensate_gravity`` (then ``tau = u + Y(q, 0, 0) theta``) and 0 without.  The
        control point, and so the path term of the cost, does not depend on ``theta``.

        Output-error identification fits ``theta`` so that the plant replays a recorded track, with no ``ddq`` (nor
        any differentiated measurement) needed.  Cut the recorded positions ``q_rec`` (``(T + 1, n)``) and applied
        torques ``u_rec`` (``(T, n)``) into ``B`` windows of ``S`` steps that start at recorded states (``dq`` at a
        window start from the record, or a free parameter), replay the recorded torques without compensation and
        compare positions::

            q0, dq0 = q_rec[starts], dq_rec[starts]                               # (B, n) window starts
            u = torch.stack([u_rec[s:s + S] for s in starts], 1)                  # (S, B, n) recorded torques
            target = torch.stack([q_rec[s + 1:s + S + 1] for s in starts], 1)     # (S, B, n)
            theta = torch.tensor(rc.inertial_parameters(), device="cuda", requires_grad=True)

            def loss():
                _, _, traj, _ = rc.simulate(q0, dq0, u, dt=dt, compensate_gravity=False, record=("q",), theta=theta)
                return (traj["q"] - target).pow(2).sum()

        and minimise ``loss`` over ``theta`` (e.g. ``torch.optim.LBFGS``; for a link's three tied masses write
        ``theta = T @ phi`` with ``arms._ident.tie_matrix(n)`` and optimise ``phi``).  Short windows keep the problem
        well conditioned; directions of ``theta`` the motion does not excite stay where they start."""
        from ..controllers import _batch

        rc = self if theta is None else self._with_theta(theta)
        if torch is not None and _is_torch(path) and path.requires_grad and torch.is_grad_enabled():
            raise NotImplementedError("simulate is not differentiable with respect to the path")
        if torch is not None and _is_torch_grad(q, dq, u, theta):
            from . import _autograd

            return _autograd.simulate(rc, q, dq, u, dt, path, effort_weight, compensate_gravity, ref_frame,
                                      xyz_offset, record, theta)
        if rc is not self:
            return rc.simulate(q, dq, u, dt=dt, path=path, effort_weight=effort_weight,
                               compensate_gravity=compensate_gravity, ref_frame=ref_frame, xyz_offset=xyz_offset,
                               record=record)
        qa, dqa, single, kind, f32 = self._on_device(q, dq)
        if kind == "torch":
            qa, dqa = qa.clone(), dqa.clone()
        B, n = qa.shape

        def rows(x, width, what):
            t = x if _is_torch(x) else torch.as_tensor(np.asarray(x, dtype=np.float64))
            t = t.to(device=qa.device, dtype=qa.dtype).contiguous()
            if t.dim() == 2 and t.shape[1] == width:
                return t, 0
            if t.dim() == 3 and t.shape[1:] == (B, width):
                return t, width
            raise ValueError(f"{what} must have shape (S, {width}) or (S, {B}, {width})")

        ua, ustride = rows(u, n, "u")
        steps = ua.shape[0]
        pth, pstride = (None, 0)
        if path is not None:
            pth, pstride = rows(path, 6, "path")
            if pth.shape[0] != steps:
                raise ValueError(f"path has {pth.shape[0]} steps, u has {steps}")
        fid = self.frame_id(ref_frame)
        xo = None
        if xyz_offset is not None and not np.allclose(np.asarray(xyz_offset, dtype=float), 0):
            xo = (C.c_double * 3)(*[float(v) for v in np.asarray(xyz_offset, dtype=float).reshape(3)])
        for k in record:
            if k not in ("q", "dq", "u", "x"):
                raise ValueError(f"simulate can record 'q', 'dq', 'u' and 'x', not {k!r}")
        traj = {k: torch.empty((steps, B, 3 if k == "x" else n), dtype=qa.dtype, device=qa.device) for k in record}
        cost = torch.empty((B,), dtype=qa.dtype, device=qa.device)
        L = _lib.lib()
        fn = L.abrb_plant_rollout_f32 if f32 else L.abrb_plant_rollout_f64
        with torch.cuda.device(qa.device):
            _lib.check(fn(self._handle, fid, xo, qa.data_ptr(), dqa.data_ptr(), ua.data_ptr(), ustride,
                          1 if compensate_gravity else 0, _batch.ptr(pth), pstride, int(steps), float(dt),
                          float(effort_weight), _batch.ptr(traj.get("q")), _batch.ptr(traj.get("dq")),
                          _batch.ptr(traj.get("u")), _batch.ptr(traj.get("x")), cost.data_ptr(), B,
                          torch.cuda.current_stream(qa.device).cuda_stream))
        if kind == "numpy":
            qa, dqa, cost = qa.cpu().numpy(), dqa.cpu().numpy(), cost.cpu().numpy()
            traj = {k: v.cpu().numpy() for k, v in traj.items()}
        if single:
            return qa[0], dqa[0], {k: v[:, 0] for k, v in traj.items()}, cost[0]
        return qa, dqa, traj, cost


def builtin_config(arm, **kwargs):
    """Config for one of the arms shipped with the reference: 'ur5', 'jaco2', 'threejoint', 'twojoint'."""
    return BaseConfig(_abi.load_arm_json(arm), ROBOT_NAME=arm, **kwargs)
