"""Velocity-profiled position and orientation paths, one path or a batch of start/target pairs per call.

Reference: controllers/path_planners/path_planner.py (``PathPlanner``), orientation.py (``match_position_path``) and
utils/transformations.py.  A path warps the position profile's shape onto start -> target, walks it at the speeds of
a velocity ramp up to ``max_velocity`` (lowered in steps of 0.1 until both ramps fit), a constant segment and a ramp
down, and SLERPs the orientation in step with the distance covered.  Rows are
``[x, y, z, dx, dy, dz, a, b, g, da, db, dg]`` (the last six only with orientations).

The planning runs on the device in two launches (include/abrb.h, abrb_path_*): ``abrb_path_plan`` sizes every path,
then, after the one host synchronisation of a call (reading the lengths back to size the output),
``abrb_path_fill_*`` writes the rows.  ``plot`` and ``verbose`` are accepted and ignored.
"""
import ctypes as C
import warnings

import numpy as np

from ... import _abi, _lib
from .. import _batch
from . import velocity_profiles

# transformations._AXES2TUPLE: (firstaxis, parity, repetition, frame)
AXES = {
    "sxyz": (0, 0, 0, 0), "sxyx": (0, 0, 1, 0), "sxzy": (0, 1, 0, 0), "sxzx": (0, 1, 1, 0),
    "syzx": (1, 0, 0, 0), "syzy": (1, 0, 1, 0), "syxz": (1, 1, 0, 0), "syxy": (1, 1, 1, 0),
    "szxy": (2, 0, 0, 0), "szxz": (2, 0, 1, 0), "szyx": (2, 1, 0, 0), "szyz": (2, 1, 1, 0),
    "rzyx": (0, 0, 0, 1), "rxyx": (0, 0, 1, 1), "ryzx": (0, 1, 0, 1), "rxzx": (0, 1, 1, 1),
    "rxzy": (1, 0, 0, 1), "ryzy": (1, 0, 1, 1), "rzxy": (1, 1, 0, 1), "ryxy": (1, 1, 1, 1),
    "ryxz": (2, 0, 0, 1), "rzxz": (2, 0, 1, 1), "rxyz": (2, 1, 0, 1), "rzyz": (2, 1, 1, 1),
}

# include/abrb.h ABRB_PATH_*: rows the reference cannot plan
REASONS = {
    -1: "start and target coincide (zero distance) or are not finite",
    -2: "target - start points exactly opposite to (1, 1, 1), so the path shape cannot be rotated onto it",
    -3: "the search for a reachable max_velocity reached 0",
    -4: "a velocity ramp has fewer than two samples (start or target velocity at or above the reachable maximum)",
    -5: "a velocity ramp or the constant segment would have 2^28 or more steps",
}


class PathPlanner:
    def __init__(self, pos_profile, vel_profile, axes="rxyz", verbose=False):
        """``pos_profile``: any object with ``step(t)`` and ``n_sample_points`` (position_profiles); ``vel_profile``:
        ``velocity_profiles.Gaussian`` or ``velocity_profiles.Linear`` (the two kinds the device evaluates)."""
        if type(vel_profile) not in (velocity_profiles.Gaussian, velocity_profiles.Linear):
            raise TypeError(f"vel_profile must be velocity_profiles.Gaussian or velocity_profiles.Linear, got "
                            f"{type(vel_profile).__name__} (the device evaluates only these two ramps)")
        if axes not in AXES:
            raise ValueError(f"unknown Euler axes {axes!r}")
        self.n_sample_points = int(pos_profile.n_sample_points)
        if not 2 <= self.n_sample_points <= _abi.PATH_MAX_POINTS:
            raise ValueError(f"n_sample_points must be in 2 .. {_abi.PATH_MAX_POINTS}")
        self.dt = vel_profile.dt
        self.pos_profile = pos_profile
        self.vel_profile = vel_profile
        self.axes = axes
        self.verbose = verbose
        # step(t_i) does not depend on the path, so the profile is sampled once per planner
        ts = np.linspace(0, 1, self.n_sample_points)
        self.table = np.ascontiguousarray([np.asarray(pos_profile.step(t), dtype=np.float64) for t in ts])
        self._dev_table = {}
        self.params = _abi.PathParams()
        self.params.vel_kind = vel_profile.KIND
        self.params.n_points = self.n_sample_points
        self.params.dt = float(vel_profile.dt)
        self.params.acceleration = float(vel_profile.acceleration)
        self.params.n_sigma = float(getattr(vel_profile, "n_sigma", 1.0))
        for i, v in enumerate(AXES[axes]):
            self.params.axes[i] = v
        self.n = 0
        self.n_timesteps = None
        self.path = np.zeros((12, 1))

    def _table_on(self, device):
        import torch

        key = str(device)
        if key not in self._dev_table:
            self._dev_table[key] = torch.as_tensor(self.table, device=device)
        return self._dev_table[key]

    def generate_path(self, start_position, target_position, max_velocity, start_orientation=None,
                      target_orientation=None, start_velocity=0, target_velocity=0, plot=False):
        """``start_position``, ``target_position`` (3,) -> path (S, 12), or (S, 6) without orientations, as the
        reference.  (B, 3) -> (B, S_max, w): rows past a path's own length ``self.lengths[b]`` repeat its last row.
        Orientations: (3,) Euler angles in the order ``axes``, or (B, 3) per path.  ``max_velocity``,
        ``start_velocity``, ``target_velocity``: scalars or (B,).  NumPy in -> NumPy out; CUDA tensors in -> CUDA
        tensors out (a view of one (S_max, B, w) buffer).  The output dtype is the position's (float64 or float32); the
        planning itself is float64 in both."""
        import torch

        # the reference's rejections (path_planner.py:144-151, 368-371), before any device work
        vh = [np.asarray(v.detach().cpu() if _batch.is_torch(v) else v, dtype=np.float64)
              for v in (max_velocity, start_velocity, target_velocity)]
        for name, v in (("start", vh[1]), ("target", vh[2])):
            bad = np.nonzero(np.ravel(~(v <= vh[0])))[0]
            if bad.size:
                vb, mb = np.broadcast_arrays(v, vh[0])
                i = bad[0]
                raise AssertionError(f"{name} velocity ({np.ravel(vb)[i]} m/s) > max velocity ({np.ravel(mb)[i]} m/s)"
                                     + ("" if vb.ndim == 0 else f" in row {i}"))
        orient = start_orientation is not None
        if orient and target_orientation is None:
            raise NotImplementedError("A target orientation is required to generate path")
        is_t = _batch.is_torch(start_position)
        single = (start_position.dim() if is_t else np.ndim(start_position)) == 1
        if is_t:
            dev = start_position.device
            if dev.type != "cuda":
                raise ValueError("torch inputs must be CUDA tensors")
            out_dtype = start_position.dtype
        else:
            dev = torch.device("cuda", torch.cuda.current_device())
            out_dtype = torch.float32 if np.asarray(start_position).dtype == np.float32 else torch.float64
        if out_dtype not in (torch.float32, torch.float64):
            raise ValueError("positions must be float32 or float64")

        def dev64(x, what, shape):
            t = x.detach() if _batch.is_torch(x) else torch.as_tensor(np.asarray(x, dtype=np.float64))
            t = t.to(device=dev, dtype=torch.float64)
            if t.shape != shape:
                try:
                    t = t.expand(shape)
                except RuntimeError:
                    raise ValueError(f"{what} must have shape {tuple(shape[1:]) or '()'} or {tuple(shape)}") from None
            return t.contiguous()

        sp = dev64(start_position, "start_position", (1, 3) if single else tuple(start_position.shape))
        if sp.dim() != 2 or sp.shape[1] != 3:
            raise ValueError("start_position must have shape (3,) or (B, 3)")
        B = sp.shape[0]
        tp = dev64(target_position, "target_position", (B, 3))
        speeds = [dev64(v, name, (B,)) for v, name in ((max_velocity, "max_velocity"),
                                                      (start_velocity, "start_velocity"),
                                                      (target_velocity, "target_velocity"))]
        vmax, v0, v1 = speeds
        so = dev64(start_orientation, "start_orientation", (B, 3)) if orient else None
        to = dev64(target_orientation, "target_orientation", (B, 3)) if orient else None
        w = 12 if orient else 6

        L = _lib.lib()
        table = self._table_on(dev)
        p = C.byref(self.params)
        lengths = torch.empty(B, dtype=torch.int64, device=dev)
        plan = torch.empty((B, C.sizeof(_abi.PathRec) // 8), dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(L.abrb_path_plan(p, table.data_ptr(), sp.data_ptr(), tp.data_ptr(), vmax.data_ptr(),
                                        v0.data_ptr(), v1.data_ptr(), lengths.data_ptr(), plan.data_ptr(), B, stream))
            lh = lengths.cpu().numpy()  # the one host synchronisation: the output's size
            bad = np.nonzero(lh < 2)[0]
            if bad.size:
                r = int(lh[bad[0]])
                raise ValueError(f"cannot plan {'the path' if single else f'row {bad[0]}'}: {REASONS.get(r, r)}")
            s_max = int(lh.max()) if B else 0
            buf = torch.empty((s_max, B, w), dtype=out_dtype, device=dev)
            fill = L.abrb_path_fill_f32 if out_dtype == torch.float32 else L.abrb_path_fill_f64
            _lib.check(fill(p, table.data_ptr(), sp.data_ptr(), tp.data_ptr(), v0.data_ptr(), v1.data_ptr(),
                            so.data_ptr() if orient else None, to.data_ptr() if orient else None, plan.data_ptr(),
                            lengths.data_ptr(), s_max, buf.data_ptr(), B, stream))
        path = buf.permute(1, 0, 2)
        if single:
            path = path[0]
        if not is_t:
            path = path.cpu().numpy()
            # the reference's check of the end point (path_planner.py:437-450), wherever the rows are on the host
            ends = path[-1, :3] if single else path[:, -1, :3]
            tgt = np.asarray(target_position, dtype=np.float64)
            err = np.linalg.norm(np.atleast_2d(ends) - np.atleast_2d(tgt), axis=-1)
            if np.any(err >= 0.01):
                warnings.warn(f"the distance at the end of the generated path to the target position is "
                              f"{float(err.max())} m; a path shape with lower frequency terms, more sample points, a "
                              f"smaller dt, or lower velocities and acceleration lower it")

        self.lengths = lengths if is_t else lh
        self.n_timesteps = s_max
        self.time_to_converge = s_max * self.dt
        self.n = 0
        self.path = path
        self.position_path = path[..., 0:3]
        self.velocity_path = path[..., 3:6]
        if orient:
            self.orientation_path = path[..., 6:9]
            self.ang_velocity_path = path[..., 9:12]
        return self.path

    def _row(self, n):
        return self.path[n] if self.path.ndim == 2 else self.path[:, n]

    def next(self):
        """The next row of the path (of every path of a batch); it stays at the last row once there."""
        row = self._row(self.n)
        if self.n_timesteps is not None:
            self.n = min(self.n + 1, self.n_timesteps - 1)
        else:
            self.n += 1
        return row

    def next_at_n(self, n):
        """Row n without moving the iterator; the last row for n past the end."""
        return self._row(min(n, self.n_timesteps - 1))
