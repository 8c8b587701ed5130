"""Sliding-mode controller (Slotine & Li).

Reference: /root/reference/abr_control/controllers/sliding.py:6-99 —
``u = M ddq_ref + C dq_ref + g - kd s`` with ``s = dq - dq_ref``; in Cartesian mode the references come from
``pinv(J[:3])`` of the position error, in joint mode from the joint error.  ``self.s`` (the signal the reference hands
to its dynamics adaptation) is stored on every call.  One state or a batch, one kernel launch per call.
"""
import ctypes as C

import numpy as np

from .. import _lib
from . import _batch
from .controller import Controller


class Sliding(Controller):
    def __init__(self, robot_config, kd=160.0, lamb=30.0, cartesian=True):
        super().__init__(robot_config)
        self.kd = kd
        self.lamb = lamb
        self.cartesian = cartesian
        self.s = None

    def generate(self, q, dq, target, target_velocity=0, target_acc=0, ref_frame="EE", offset=None):
        import torch

        rc = self.robot_config
        n = rc.N_JOINTS
        w = 3 if self.cartesian else n
        qa, dqa, single, kind, f32 = _batch.prep_state(rc, q, dq)
        B = qa.shape[0]

        def rows(x, what):
            if x is None or (np.isscalar(x) and x == 0):
                return None, 0
            if np.isscalar(x):
                x = np.full(w, float(x))
            return _batch.prep_rows(x, qa, kind, w, what)

        tgt, ts = _batch.prep_rows(target, qa, kind, w, "target")
        tv, tvs = rows(target_velocity, "target_velocity")
        ta, tas = rows(target_acc, "target_acc")
        xo = None
        if offset is not None and not np.allclose(np.asarray(offset, dtype=float), 0):
            xo = (C.c_double * 3)(*[float(v) for v in np.asarray(offset, dtype=float).reshape(3)])
        fid = rc.frame_id(ref_frame)
        arrays = [qa, dqa, tgt, tv, ta]
        if kind == "numpy":
            dev = torch.device("cuda", torch.cuda.current_device())
            arrays = [None if a is None else torch.as_tensor(a).to(dev) for a in arrays]
        tq = arrays[0]
        u, s = torch.empty_like(tq), torch.empty_like(tq)
        L = _lib.lib()
        fn = L.abrb_sliding_generate_f32 if f32 else L.abrb_sliding_generate_f64
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        with torch.cuda.device(tq.device):
            _lib.check(fn(rc.handle, float(self.kd), float(self.lamb), int(bool(self.cartesian)), fid, xo, ptr(arrays[0]),
                          ptr(arrays[1]), ptr(arrays[2]), ts, ptr(arrays[3]), tvs, ptr(arrays[4]), tas, u.data_ptr(),
                          s.data_ptr(), B, torch.cuda.current_stream(tq.device).cuda_stream))
        if kind == "numpy":
            u, s = u.cpu().numpy(), s.cpu().numpy()
            self.s = np.array(s[0], dtype=np.float64) if single else s
            return np.array(u[0], dtype=np.float64) if single else u
        self.s = s[0] if single else s
        return u[0] if single else u

    def rollout_path(self, q, dq, path, dt=1e-3, path_velocity=None, path_acc=None, ref_frame="EE", offset=None,
                     record=("q", "dq", "u", "x"), effort_weight=0.0):
        """Closed-loop rollout of this controller along a path on the GPU (include/abrb.h,
        abrb_sliding_rollout_path_*): for each step ``t = 0 .. S-1``::

            u_t = generate(q_t, dq_t, path[t], path_velocity[t], path_acc[t], ref_frame, offset)
            x_t = Tx(ref_frame, q_t, x=offset)
            ddq = M^-1 (u_t + g - C dq_t);  dq_{t+1} = dq_t + ddq dt;  q_{t+1} = q_t + dq_{t+1} dt
            cost += e_t + effort_weight * |u_t|^2

        with the error the controller drives to zero: ``e_t = |x_t - path[t]|^2`` in Cartesian mode and
        ``|q_t - path[t]|^2`` (not wrapped, as the reference's joint-mode error) in joint mode, where ``ref_frame``
        and ``offset`` only choose the recorded ``x``.  ``path``, ``path_velocity`` and ``path_acc`` (None: zero) have
        rows of 3 values (Cartesian) or n (joint mode), ``(S, w)`` shared by every trajectory or ``(S, B, w)``.

        Gravity: ``generate`` adds ``+g`` as the reference does (sliding.py:97), while the plant is held still by
        ``u = -g``; so on an arm with gravity the closed loop runs against a ``2 g`` bias.  The rollout reproduces
        ``generate`` as it is.

        Returns ``(q_final, dq_final, traj, cost)`` as ``OSC.rollout_path`` (records ``"q"``, ``"dq"``, ``"u"``:
        ``(S, B, n)``, ``"x"``: ``(S, B, 3)``; ``u`` and ``x`` of the state before step t, ``q`` and ``dq`` after it;
        ``record=()`` for the cost only), in the input's form (CUDA tensors or NumPy; a single ``(n,)`` state takes an
        ``(S, w)`` path).  ``q``, ``dq`` and ``self.s`` are left as they are."""
        rc = self.robot_config
        w = 3 if self.cartesian else rc.N_JOINTS
        gains = (float(self.kd), float(self.lamb), int(bool(self.cartesian)))
        return _batch.ctrl_rollout(rc, ("abrb_sliding_rollout_path_f64", "abrb_sliding_rollout_path_f32"), gains, q,
                                   dq, [(path, "path"), (path_velocity, "path_velocity"), (path_acc, "path_acc")], w,
                                   dt, ref_frame, offset, record, effort_weight, "rollout_path")
