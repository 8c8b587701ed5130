"""Velocity ramps of a planned path, as the reference's ``path_planners.velocity_profiles``.

``generate`` is the host (NumPy) form of a ramp, kept for parity checks.  ``PathPlanner`` never calls it: the device
evaluates exactly these two kinds from ``KIND`` and the parameters (abrb_path.cuh, ``ramp_at``).
"""
import numpy as np

from ... import _abi


class VelProf:
    def __init__(self, dt):
        self.dt = dt

    def generate(self, start_velocity, target_velocity):
        raise NotImplementedError


class Gaussian(VelProf):
    """Left half of a Gaussian over ``n_sigma`` standard deviations, shifted to start at ``start_velocity`` and scaled to
    end at ``target_velocity``; ``int((target - start) / acceleration / dt)`` samples."""

    KIND = _abi.VEL_GAUSSIAN

    def __init__(self, dt, acceleration, n_sigma=3):
        self.acceleration = acceleration
        self.n_sigma = n_sigma
        super().__init__(dt=dt)

    def generate(self, start_velocity, target_velocity):
        dv = target_velocity - start_velocity
        n = int(dv / self.acceleration / self.dt)
        s = 1 / (dv * np.sqrt(np.pi * 2))
        u = self.n_sigma * s
        x = np.linspace(0, u, n)
        v = 1 * (1 / (s * np.sqrt(2 * np.pi)) * np.exp(-0.5 * ((x - u) / s) ** 2))
        v -= v[0]
        v *= dv / v[-1]
        v += start_velocity
        return v


class Linear(VelProf):
    """Straight ramp from ``start_velocity`` to ``target_velocity`` with slope ``acceleration``."""

    KIND = _abi.VEL_LINEAR

    def __init__(self, dt, acceleration):
        self.acceleration = acceleration
        super().__init__(dt=dt)

    def generate(self, start_velocity, target_velocity):
        steps = (target_velocity - start_velocity) / self.acceleration / self.dt
        return np.linspace(start_velocity, target_velocity, int(steps))
