"""Joint-space PD controller.

Reference: /root/reference/abr_control/controllers/joint.py:6-131 —
``u = M (kp q_tilde + kv (target_velocity - dq)) - g`` with ``q_tilde = ((target - q + pi) mod 2 pi) - pi``.
The ball-joint (quaternion) branch of the reference (joint.py:48-102) exists only for MuJoCo models and is not built.
One state or a batch (NumPy host buffers or CUDA tensors), one kernel launch per call.
"""
import numpy as np

from .. import _lib
from . import _batch
from .controller import Controller


def _device_call(rc, fn_f32, fn_f64, head_args, arrays, single):
    """shared plumbing: arrays = [(array or None)...] already (B, w) contiguous, first one is q."""
    import torch

    q = arrays[0]
    kind = "torch" if _batch.is_torch(q) else "numpy"
    if kind == "numpy":
        dev = torch.device("cuda", torch.cuda.current_device())
        arrays = [None if a is None else torch.as_tensor(a).to(dev) for a in arrays]
        q = arrays[0]
    f32 = q.dtype == torch.float32
    u = torch.empty_like(q)
    fn = fn_f32 if f32 else fn_f64
    with torch.cuda.device(q.device):
        _lib.check(fn(*head_args(arrays, u), torch.cuda.current_stream(q.device).cuda_stream))
    if kind == "numpy":
        u = u.cpu().numpy()
        return np.array(u[0], dtype=np.float64) if single else u
    return u[0] if single else u


class Joint(Controller):
    def __init__(self, robot_config, kp=1, kv=None, quaternions=None, account_for_gravity=True):
        if quaternions is not None:
            raise NotImplementedError("ball-joint (quaternion) states are a MuJoCo-only branch of the reference")
        super().__init__(robot_config)
        self.kp = kp
        self.kv = np.sqrt(self.kp) if kv is None else kv
        self.account_for_gravity = account_for_gravity
        self.ZEROS_N_JOINTS = np.zeros(robot_config.N_JOINTS)

    def generate(self, q, dq, target, target_velocity=None):
        rc = self.robot_config
        n = rc.N_JOINTS
        qa, dqa, single, kind, _ = _batch.prep_state(rc, q, dq)
        tgt, tstride = _batch.prep_rows(target, qa, kind, n, "target")
        tv, tvstride = (None, 0)
        if target_velocity is not None:
            tv, tvstride = _batch.prep_rows(target_velocity, qa, kind, n, "target_velocity")
        L = _lib.lib()
        B = qa.shape[0]

        def args(a, u):
            return (rc.handle, float(self.kp), float(self.kv), int(bool(self.account_for_gravity)), a[0].data_ptr(),
                    a[1].data_ptr(), a[2].data_ptr(), tstride, None if a[3] is None else a[3].data_ptr(), tvstride,
                    u.data_ptr(), B)

        return _device_call(rc, L.abrb_joint_generate_f32, L.abrb_joint_generate_f64, args, [qa, dqa, tgt, tv], single)

    def rollout_path(self, q, dq, path, dt=1e-3, path_velocity=None, ref_frame="EE", xyz_offset=None,
                     record=("q", "dq", "u", "x"), effort_weight=0.0):
        """Closed-loop rollout of this controller along a joint-space path on the GPU (include/abrb.h,
        abrb_joint_rollout_path_*): for each step ``t = 0 .. S-1``::

            u_t = generate(q_t, dq_t, target=path[t], target_velocity=path_velocity[t])
            x_t = Tx(ref_frame, q_t, x=xyz_offset)
            ddq = M^-1 (u_t + g - C dq_t);  dq_{t+1} = dq_t + ddq dt;  q_{t+1} = q_t + dq_{t+1} dt
            cost += |wrap(path[t] - q_t)|^2 + effort_weight * |u_t|^2        (wrap: into [-pi, pi), as generate)

        ``path`` and ``path_velocity`` (rad/s; None: zero) are ``(S, n)`` (shared by every trajectory) or ``(S, B,
        n)``.  Returns ``(q_final, dq_final, traj, cost)`` as ``OSC.rollout_path``: ``traj[k]`` for k in ``record`` is
        ``(S, B, n)`` (``"x"``: ``(S, B, 3)``); ``traj["u"][t]`` and ``traj["x"][t]`` belong to the state before step
        t, ``traj["q"][t]`` and ``traj["dq"][t]`` to the state after it; ``cost`` is ``(B,)``; ``record=()`` gives the
        final state and the cost only.  CUDA tensors in -> CUDA tensors out; NumPy in -> NumPy out; a single state
        ``(n,)`` takes an ``(S, n)`` path and returns ``(S, .)`` records and a scalar cost.  ``q`` and ``dq`` are not
        modified.  The plant is that of ``simulate``, so ``traj["u"]`` replayed there gives back the track.

        Tracking joint paths planned by ``InverseKinematics.generate_path`` for a batch of starts: its ``(B, S, n)``
        position path is a view of one ``(S, B, n)`` buffer, so ``permute`` hands it over without a copy.  The
        planner's velocity path is the joint step of each iteration, not a velocity in rad/s, so it is not a
        ``path_velocity``::

            pos, _ = ik.generate_path(q0, targets, n_timesteps=S)          # (B, S, n)
            qf, dqf, tr, cost = Joint(rc, kp=300, kv=20).rollout_path(q0, dq0, pos.permute(1, 0, 2))
        """
        rc = self.robot_config
        n = rc.N_JOINTS
        gains = (float(self.kp), float(self.kv), int(bool(self.account_for_gravity)))
        return _batch.ctrl_rollout(rc, ("abrb_joint_rollout_path_f64", "abrb_joint_rollout_path_f32"), gains, q, dq,
                                   [(path, "path"), (path_velocity, "path_velocity")], n, dt, ref_frame, xyz_offset,
                                   record, effort_weight, "rollout_path")
