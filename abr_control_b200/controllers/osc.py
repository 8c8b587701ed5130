"""Batched operational-space controller.

Same constructor and ``generate`` signature as ``abr_control.controllers.OSC``
(/root/reference/abr_control/controllers/osc.py:53-66 and :217-219).  ``generate`` accepts one state
(``q`` of shape ``(n,)`` -> fresh writable float64 ``(n,)`` array, like the reference) or a batch
(``(B, n)`` NumPy -> NumPy, CUDA tensor -> CUDA tensor).  One call is one fused kernel launch:
chain walk, J / M / g / C dq, Cholesky of M, task-space inertia with the reference's det-threshold / pinv
branch (osc.py:120-147), task PD with optional velocity limiting (osc.py:198-215), orientation error by either
algorithm (osc.py:149-196), gravity / Coriolis compensation and the null-space filter for the secondary
controllers (osc.py:310-318).

``ki != 0`` (osc.py:81-82, :262-264): the reference keeps ONE ``integrated_error`` vector per controller because it
evaluates one state per call.  Here a single-state call keeps exactly that (``self.integrated_error``, shape ``(6,)``);
a batched call keeps one integrator row per state in a ``(B, 6)`` buffer owned by the controller and reused by every
later call with the same batch shape / dtype / device (``integrated_error_batch``); ``reset_integrated_error()`` zeroes
both.
"""
import ctypes as C

import numpy as np

from .. import _abi, _lib
from . import _batch
from ._null import NullController
from .controller import Controller


class OSC(Controller):
    def __init__(
        self,
        robot_config,
        kp=1,
        ko=None,
        kv=None,
        ki=0,
        vmax=None,
        ctrlr_dof=None,
        null_controllers=None,
        use_g=True,
        use_C=False,
        orientation_algorithm=0,
    ):
        super().__init__(robot_config)
        self.kp = kp
        self.ko = kp if ko is None else ko
        self.kv = np.sqrt(self.kp + self.ko) if kv is None else kv
        self.ki = ki
        self.null_controllers = null_controllers
        self.use_g = use_g
        self.use_C = use_C
        self.orientation_algorithm = orientation_algorithm
        if self.ki != 0:
            self.integrated_error = np.zeros(6)
        self._ierr_batch = {}
        if ctrlr_dof is None:
            ctrlr_dof = [True, True, True, False, False, False]
        self.ctrlr_dof = np.copy(ctrlr_dof)
        self.n_ctrlr_dof = np.sum(self.ctrlr_dof)
        self.task_space_gains = np.array([self.kp] * 3 + [self.ko] * 3)
        self.lamb = self.task_space_gains / self.kv
        if self.n_ctrlr_dof > robot_config.N_JOINTS:
            print(
                f"\nRobot has fewer DOF ({robot_config.N_JOINTS}) than the specified number of "
                f"space dimensions to control ({self.n_ctrlr_dof}), Poor performance may result.\n"
            )
        self.vmax = vmax
        if vmax is not None:
            self.sat_gain_xyz = vmax[0] / self.kp * self.kv
            self.sat_gain_abg = vmax[1] / self.ko * self.kv
            self.scale_xyz = vmax[0] / self.kp * self.kv
            self.scale_abg = vmax[1] / self.ko * self.kv
        if self.orientation_algorithm not in (0, 1):
            raise Exception(
                f"Invalid algorithm number {self.orientation_algorithm} for calculating orientation error"
            )
        for nc in self.null_controllers or []:
            if not isinstance(nc, NullController):
                raise TypeError("null_controllers must be abr_control_b200 Damping / RestingConfig / AvoidObstacles")
            nc._owners.add(self)
        self.training_signal = None
        # the reference stores `training_signal` on every call (osc.py:297); for large host batches it doubles the
        # device-to-host traffic, so throughput-minded callers may switch it off
        self.record_training_signal = True
        self._options = {}
        self._handle = None

    # ------------------------------------------------------------------ native handle
    # attributes baked into the native handle: the reference reads them on every call, so a later write
    # (ctrlr.use_g = False, ctrlr.kv = ...) must take effect here too -> the handle is rebuilt on the next call
    _PARAMS = frozenset(("kp", "ko", "kv", "ki", "vmax", "ctrlr_dof", "null_controllers", "use_g", "use_C",
                         "orientation_algorithm"))

    def __setattr__(self, name, value):
        if name in OSC._PARAMS and self.__dict__.get("_handle") is not None:
            self._invalidate()
        object.__setattr__(self, name, value)

    def _invalidate(self):
        if self._handle is not None:
            _lib.lib().abrb_osc_destroy(self._handle)
            self._handle = None

    def _native(self):
        if self._handle is None:
            n = self.robot_config.N_JOINTS
            nulls = [nc._params() for nc in (self.null_controllers or [])]
            p = _abi.osc_params(
                n, kp=self.kp, ko=self.ko, kv=self.kv, ki=self.ki, vmax=self.vmax, ctrlr_dof=list(self.ctrlr_dof),
                null=nulls, use_g=self.use_g, use_C=self.use_C, orientation_algorithm=self.orientation_algorithm,
            )
            h = C.c_void_p()
            _lib.check(_lib.lib().abrb_osc_create(self.robot_config.handle, C.byref(p), C.byref(h)))
            self._handle = h
            for name, value in self._options.items():
                _lib.check(_lib.lib().abrb_osc_set_option(h, name.encode(), value))
        return self._handle

    def set_option(self, name, value):
        """Execution option of the native controller (include/abrb.h, abrb_osc_set_option), e.g.
        ``set_option("host_chunk_states", 32768)``.  Kept across parameter changes."""
        self._options[name] = float(value)
        if self._handle is not None:
            _lib.check(_lib.lib().abrb_osc_set_option(self._handle, name.encode(), float(value)))

    def __del__(self):
        try:
            self._invalidate()
        except Exception:
            pass

    # ------------------------------------------------------------------ integrator state (ki != 0)
    def reset_integrated_error(self):
        if self.ki != 0:
            self.integrated_error = np.zeros(6)
        for buf in self._ierr_batch.values():
            buf.zero_() if _batch.is_torch(buf) else buf.fill(0)

    def _ierr_for(self, like, kind, single):
        """the (B, 6) integrator buffer for this call's batch (None when ki == 0)"""
        if self.ki == 0:
            return None
        if single:
            one = np.asarray(self.integrated_error, dtype=np.float64).reshape(1, 6)
            if kind == "torch":
                import torch

                return torch.as_tensor(one).to(device=like.device, dtype=like.dtype)
            return np.ascontiguousarray(one.astype(like.dtype))
        key = (kind, like.shape[0], str(like.dtype), str(like.device) if kind == "torch" else "host")
        buf = self._ierr_batch.get(key)
        if buf is None:
            if kind == "torch":
                import torch

                buf = torch.zeros((like.shape[0], 6), dtype=like.dtype, device=like.device)
            else:
                buf = _batch.host_out((like.shape[0], 6), like.dtype)
                buf.fill(0)
            self._ierr_batch[key] = buf
        return buf

    @property
    def integrated_error_batch(self):
        """{(kind, B, dtype, device): (B, 6) buffer} of the batched calls made so far"""
        return self._ierr_batch

    # ------------------------------------------------------------------ generate
    def _call_args(self, q, dq, target, target_velocity, ref_frame, xyz_offset):
        rc = self.robot_config
        qa, dqa, single, kind, f32 = _batch.prep_state(rc, q, dq)
        tgt, tstride = _batch.prep_rows(target, qa, kind, 6, "target")
        tv, tvstride = (None, 0)
        if target_velocity is not None:
            tv, tvstride = _batch.prep_rows(target_velocity, qa, kind, 6, "target_velocity")
        fid = rc.frame_id(ref_frame)
        xo = None
        if xyz_offset is not None and not np.allclose(np.asarray(xyz_offset, dtype=float), 0):
            xo = (C.c_double * 3)(*[float(v) for v in np.asarray(xyz_offset, dtype=float).reshape(3)])
        return qa, dqa, single, kind, f32, tgt, tstride, tv, tvstride, fid, xo

    def generate(self, q, dq, target, target_velocity=None, ref_frame="EE", xyz_offset=None):
        qa, dqa, single, kind, f32, tgt, tstride, tv, tvstride, fid, xo = self._call_args(
            q, dq, target, target_velocity, ref_frame, xyz_offset)
        B = qa.shape[0]
        L = _lib.lib()
        h = self._native()
        ie = self._ierr_for(qa, kind, single)
        if kind == "torch":
            import torch

            with torch.cuda.device(qa.device):
                u = torch.empty_like(qa)
                tr = torch.empty_like(qa)
                fn = L.abrb_osc_generate_f32 if f32 else L.abrb_osc_generate_f64
                _lib.check(fn(h, fid, xo, qa.data_ptr(), dqa.data_ptr(), tgt.data_ptr(), tstride, _batch.ptr(tv),
                              tvstride, u.data_ptr(), tr.data_ptr(), _batch.ptr(ie), B,
                              torch.cuda.current_stream(qa.device).cuda_stream))
        else:
            u = _batch.host_out(qa.shape, qa.dtype)
            tr = _batch.host_out(qa.shape, qa.dtype) if (self.record_training_signal or single) else None
            fn = L.abrb_osc_generate_host_f32 if f32 else L.abrb_osc_generate_host_f64
            _lib.check(fn(h, fid, xo, qa.ctypes.data, dqa.ctypes.data, tgt.ctypes.data, tstride, _batch.ptr(tv),
                          tvstride, u.ctypes.data, _batch.ptr(tr), _batch.ptr(ie), B))
        if single:
            if ie is not None:
                self.integrated_error = np.array(ie[0].cpu() if kind == "torch" else ie[0], dtype=np.float64)
            self.training_signal = np.array(tr[0], dtype=np.float64) if kind == "numpy" else tr[0]
            return np.array(u[0], dtype=np.float64) if kind == "numpy" else u[0]
        self.training_signal = tr
        return u

    def generate_async(self, q, dq, target, target_velocity=None, ref_frame="EE", xyz_offset=None, slot=0):
        """Batched ``generate`` on HOST arrays that returns before the GPU has finished (include/abrb.h,
        abrb_osc_generate_host_async_*): the call enqueues H2D copies, kernel and D2H copies on pipeline slot ``slot``
        (0 or 1) and returns a handle whose ``wait()`` gives ``u``.  Alternating the two slots lets batch k+1's upload
        run under batch k's kernel and download.  Inputs should be page-locked (``torch.Tensor.pin_memory().numpy()``)
        and must not be modified before ``wait()``; the training signal is recorded when
        ``record_training_signal`` is set and lands in ``self.training_signal`` at ``wait()``."""
        qa, dqa, single, kind, f32, tgt, tstride, tv, tvstride, fid, xo = self._call_args(
            q, dq, target, target_velocity, ref_frame, xyz_offset)
        if kind != "numpy" or single:
            raise ValueError("generate_async takes batched host (NumPy) arrays; CUDA tensors are asynchronous already")
        L = _lib.lib()
        h = self._native()
        ie = self._ierr_for(qa, kind, False)
        u = _batch.host_out(qa.shape, qa.dtype)
        tr = _batch.host_out(qa.shape, qa.dtype) if self.record_training_signal else None
        fn = L.abrb_osc_generate_host_async_f32 if f32 else L.abrb_osc_generate_host_async_f64
        _lib.check(fn(h, fid, xo, qa.ctypes.data, dqa.ctypes.data, tgt.ctypes.data, tstride, _batch.ptr(tv), tvstride,
                      u.ctypes.data, _batch.ptr(tr), _batch.ptr(ie), qa.shape[0], int(slot)))
        return _Pending(self, int(slot), u, tr, (qa, dqa, tgt, tv, ie))

    def generate_into(self, q, dq, target, u_out, training_out=None, target_velocity=None, ref_frame="EE",
                      xyz_offset=None, integrated_error=None):
        """Allocation-free batched ``generate`` for hot loops: all arguments are contiguous CUDA tensors of one dtype
        (``q, dq, u_out, training_out``: (B, n); ``target, target_velocity``: (B, 6) or (6,); ``integrated_error``:
        (B, 6), required iff ki != 0); the result is written into ``u_out`` on the current torch stream of the
        tensors' device.  No shape massaging, one ctypes call."""
        import torch

        rc = self.robot_config
        B, n = q.shape
        if n != rc.N_JOINTS or dq.shape != q.shape or u_out.shape != q.shape or not q.is_cuda:
            raise ValueError("generate_into: q, dq, u_out must be CUDA tensors of shape (B, n_joints)")
        f32 = q.dtype == torch.float32
        for t in (dq, target, u_out, training_out, target_velocity, integrated_error):
            if t is not None and (t.dtype != q.dtype or not t.is_contiguous() or t.device != q.device):
                raise ValueError("generate_into: tensors must share dtype/device and be contiguous")
        for t, what in ((target, "target"), (target_velocity, "target_velocity")):
            if t is not None and tuple(t.shape) not in ((6,), (B, 6)):
                raise ValueError(f"generate_into: {what} must have shape (6,) or ({B}, 6)")
        if training_out is not None and training_out.shape != q.shape:
            raise ValueError("generate_into: training_out must have the shape of q")
        if (self.ki != 0) != (integrated_error is not None) or (integrated_error is not None and tuple(integrated_error.shape) != (B, 6)):
            raise ValueError(f"generate_into: integrated_error of shape ({B}, 6) is required if and only if ki != 0")
        L = _lib.lib()
        fn = L.abrb_osc_generate_f32 if f32 else L.abrb_osc_generate_f64
        xo = None
        if xyz_offset is not None:
            xo = (C.c_double * 3)(*[float(v) for v in xyz_offset])
        with torch.cuda.device(q.device):
            _lib.check(fn(self._native(), rc.frame_id(ref_frame), xo, q.data_ptr(), dq.data_ptr(), target.data_ptr(),
                          6 if target.dim() == 2 else 0, None if target_velocity is None else target_velocity.data_ptr(),
                          0 if target_velocity is None or target_velocity.dim() == 1 else 6, u_out.data_ptr(),
                          None if training_out is None else training_out.data_ptr(), _batch.ptr(integrated_error), B,
                          torch.cuda.current_stream(q.device).cuda_stream))
        return u_out

    def _generate_gather(self, q, dq, target, gather_handle, buffer_index, row0, u_out=None, target_velocity=None,
                         ref_frame="EE", xyz_offset=None):
        """``generate_into`` whose rows also land in every rank's gathered array (parallel.PeerGather)."""
        import torch

        rc = self.robot_config
        B, n = q.shape
        if n != rc.N_JOINTS or dq.shape != q.shape or not q.is_cuda or (u_out is not None and u_out.shape != q.shape):
            raise ValueError("generate (gather): q, dq[, u_out] must be CUDA tensors of shape (B, n_joints)")
        for t in (dq, target, u_out, target_velocity):
            if t is not None and (t.dtype != q.dtype or not t.is_contiguous() or t.device != q.device):
                raise ValueError("generate (gather): tensors must share dtype/device and be contiguous")
        if tuple(target.shape) not in ((6,), (B, 6)):
            raise ValueError(f"generate (gather): target must have shape (6,) or ({B}, 6)")
        if self.ki != 0:
            raise NotImplementedError("the gathered variant does not carry integrator state")
        L = _lib.lib()
        fn = L.abrb_osc_generate_gather_f32 if q.dtype == torch.float32 else L.abrb_osc_generate_gather_f64
        xo = None
        if xyz_offset is not None:
            xo = (C.c_double * 3)(*[float(v) for v in xyz_offset])
        with torch.cuda.device(q.device):
            _lib.check(fn(self._native(), rc.frame_id(ref_frame), xo, q.data_ptr(), dq.data_ptr(), target.data_ptr(),
                          6 if target.dim() == 2 else 0, None if target_velocity is None else target_velocity.data_ptr(),
                          0 if target_velocity is None or target_velocity.dim() == 1 else 6, _batch.ptr(u_out), None,
                          None, B, gather_handle, int(buffer_index), int(row0),
                          torch.cuda.current_stream(q.device).cuda_stream))

    def rollout(self, q, dq, target, steps, dt=1e-3, ref_frame="EE", xyz_offset=None, record=("q", "dq", "u")):
        """Closed-loop rollout on the GPU (SURVEY.md S8d config 4): ``steps`` iterations of
        ``u = generate(q, dq, target); ddq = M^-1 (u + g - C dq); dq += ddq dt; q += dq dt``
        (semi-implicit Euler, as /root/reference/abr_control/arms/twojoint/arm_sim.py:131-132).

        Returns ``(q_final, dq_final, traj)`` with ``traj[k]`` of shape ``(steps, B, n)`` for k in ``record``.
        CUDA tensors in -> CUDA tensors out; NumPy in -> NumPy out (staged through the current CUDA device).
        """
        import torch

        rc = self.robot_config
        qa, dqa, single, kind, f32 = _batch.prep_state(rc, q, dq)
        if kind == "numpy":
            dev = torch.device("cuda", torch.cuda.current_device())
            qa, dqa = torch.as_tensor(qa).to(dev), torch.as_tensor(dqa).to(dev)
        else:
            qa, dqa = qa.clone(), dqa.clone()
        tgt, tstride = _batch.prep_rows(target, qa, "torch", 6, "target")
        B, n = qa.shape
        fid = rc.frame_id(ref_frame)
        xo = None
        if xyz_offset is not None and not np.allclose(np.asarray(xyz_offset, dtype=float), 0):
            xo = (C.c_double * 3)(*[float(v) for v in np.asarray(xyz_offset, dtype=float).reshape(3)])
        traj = {k: torch.empty((steps, B, n), dtype=qa.dtype, device=qa.device) for k in record}
        ie = None
        if self.ki != 0:  # the rollout starts from the controller's integrator state and leaves it updated
            ie = self._ierr_for(qa, "torch", single)
        L = _lib.lib()
        fn = L.abrb_osc_rollout_f32 if f32 else L.abrb_osc_rollout_f64
        with torch.cuda.device(qa.device):
            _lib.check(fn(self._native(), fid, xo, qa.data_ptr(), dqa.data_ptr(), tgt.data_ptr(), tstride, int(steps),
                          float(dt), _batch.ptr(traj.get("q")), _batch.ptr(traj.get("dq")), _batch.ptr(traj.get("u")),
                          _batch.ptr(ie), B, torch.cuda.current_stream(qa.device).cuda_stream))
        if ie is not None and single:
            self.integrated_error = ie[0].double().cpu().numpy()
        if kind == "numpy":
            qa, dqa = qa.cpu().numpy(), dqa.cpu().numpy()
            traj = {k: v.cpu().numpy() for k, v in traj.items()}
        if single:
            return qa[0], dqa[0], {k: v[:, 0] for k, v in traj.items()}
        return qa, dqa, traj

    def rollout_path(self, q, dq, path, dt=1e-3, path_velocity=None, ref_frame="EE", xyz_offset=None,
                     record=("q", "dq", "u", "x"), effort_weight=0.0):
        """Path-following closed-loop rollout on the GPU (include/abrb.h, abrb_osc_rollout_path_*): for each step
        ``t = 0 .. S-1``::

            x_t = Tx(ref_frame, q_t, x=xyz_offset)
            u_t = generate(q_t, dq_t, target=path[t], target_velocity=path_velocity[t])
            ddq = M^-1 (u_t + g - C dq_t);  dq_{t+1} = dq_t + ddq dt;  q_{t+1} = q_t + dq_{t+1} dt
            cost += |x_t - path[t, :3]|^2 + effort_weight * |u_t|^2

        ``path`` and ``path_velocity`` are ``(S, 6)`` (one path shared by every trajectory) or ``(S, B, 6)`` (one per
        trajectory); each row is (x, y, z, Euler a, b, g) like ``generate``'s target.  A velocity row that is all zero
        (or no ``path_velocity``) gives ``generate``'s -kv M dq damping.  From a reference ``PathPlanner`` result
        ``P = planner.generate_path(...)`` (rows: position, velocity, orientation, angular velocity)::

            path = np.hstack([P[:, :3], P[:, 6:9]]);  path_velocity = np.hstack([P[:, 3:6], P[:, 9:12]])

        Returns ``(q_final, dq_final, traj, cost)``: ``traj[k]`` for k in ``record`` is ``(S, B, n)`` (``"x"``:
        ``(S, B, 3)``), ``cost`` is ``(B,)``.  ``traj["x"][t]`` and ``traj["u"][t]`` belong to the state before step t,
        ``traj["q"][t]`` and ``traj["dq"][t]`` to the state after it (as in ``rollout``).  ``record=()`` returns only the
        final state and the cost: the allocation-light form for sampling-based MPC.  CUDA tensors in -> CUDA tensors
        out; NumPy in -> NumPy out; a single state ``q`` of shape ``(n,)`` takes an ``(S, 6)`` path and returns
        ``(S, n)`` records and a scalar cost.  With ``ki != 0`` the rollout starts from the controller's integrator
        state and leaves it updated, as ``rollout`` does.
        """
        import torch

        rc = self.robot_config
        qa, dqa, single, kind, f32 = _batch.prep_state(rc, q, dq)
        if kind == "numpy":
            dev = torch.device("cuda", torch.cuda.current_device())
            qa, dqa = torch.as_tensor(qa).to(dev), torch.as_tensor(dqa).to(dev)
        else:
            qa, dqa = qa.clone(), dqa.clone()
        B, n = qa.shape

        def rows(x, what):
            t = x if _batch.is_torch(x) else torch.as_tensor(np.asarray(x, dtype=np.float64))
            t = t.to(device=qa.device, dtype=qa.dtype).contiguous()
            if t.dim() == 2 and t.shape[1] == 6:
                return t, 0
            if t.dim() == 3 and t.shape[1:] == (B, 6):
                return t, 6
            raise ValueError(f"{what} must have shape (S, 6) or (S, {B}, 6)")

        pth, pstride = rows(path, "path")
        steps = pth.shape[0]
        pv, pvstride = (None, 0)
        if path_velocity is not None:
            pv, pvstride = rows(path_velocity, "path_velocity")
            if pv.shape[0] != steps:
                raise ValueError(f"path_velocity has {pv.shape[0]} steps, path has {steps}")
        fid = rc.frame_id(ref_frame)
        xo = None
        if xyz_offset is not None and not np.allclose(np.asarray(xyz_offset, dtype=float), 0):
            xo = (C.c_double * 3)(*[float(v) for v in np.asarray(xyz_offset, dtype=float).reshape(3)])
        for k in record:
            if k not in ("q", "dq", "u", "x"):
                raise ValueError(f"rollout_path can record 'q', 'dq', 'u' and 'x', not {k!r}")
        traj = {k: torch.empty((steps, B, 3 if k == "x" else n), dtype=qa.dtype, device=qa.device) for k in record}
        cost = torch.empty((B,), dtype=qa.dtype, device=qa.device)
        ie = None
        if self.ki != 0:
            ie = self._ierr_for(qa, "torch", single)
        L = _lib.lib()
        fn = L.abrb_osc_rollout_path_f32 if f32 else L.abrb_osc_rollout_path_f64
        with torch.cuda.device(qa.device):
            _lib.check(fn(self._native(), fid, xo, qa.data_ptr(), dqa.data_ptr(), pth.data_ptr(), pstride,
                          _batch.ptr(pv), pvstride, int(steps), float(dt), float(effort_weight),
                          _batch.ptr(traj.get("q")), _batch.ptr(traj.get("dq")), _batch.ptr(traj.get("u")),
                          _batch.ptr(traj.get("x")), cost.data_ptr(), _batch.ptr(ie), B,
                          torch.cuda.current_stream(qa.device).cuda_stream))
        if ie is not None and single:
            self.integrated_error = ie[0].double().cpu().numpy()
        if kind == "numpy":
            qa, dqa, cost = qa.cpu().numpy(), dqa.cpu().numpy(), cost.cpu().numpy()
            traj = {k: v.cpu().numpy() for k, v in traj.items()}
        if single:
            return qa[0], dqa[0], {k: v[:, 0] for k, v in traj.items()}, cost[0]
        return qa, dqa, traj, cost


class _Pending:
    """Result of ``OSC.generate_async``: ``wait()`` blocks until the batch has left the GPU and returns ``u``."""

    def __init__(self, ctrlr, slot, u, tr, keep):
        self._ctrlr, self._slot, self._u, self._tr, self._keep = ctrlr, slot, u, tr, keep
        self._done = False

    def wait(self):
        if not self._done:
            _lib.check(_lib.lib().abrb_osc_host_wait(self._ctrlr._native(), self._slot))
            self._done = True
            self._keep = None
            if self._tr is not None:
                self._ctrlr.training_signal = self._tr
        return self._u
