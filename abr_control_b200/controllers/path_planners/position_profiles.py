"""Shapes of a planned path: ``step(t)`` maps t in [0, 1] to a point, from [0, 0, 0] at t = 0 to [1, 1, 1] at t = 1.

Same classes, constructors and defaults as the reference's ``path_planners.position_profiles``.  ``PathPlanner`` samples
``step`` at ``linspace(0, 1, n_sample_points)`` once and hands the table to the device, so any object with ``step(t)``
and ``n_sample_points`` works as a profile.
"""
import numpy as np


class PosProf:
    def __init__(self, tol=1e-6, n_sample_points=1000, **kwargs):
        """Checks that the profile starts at [0, 0, 0] and ends at [1, 1, 1] within ``tol``."""
        self.n_sample_points = n_sample_points
        s0 = np.asarray(self.step(0))
        assert np.sum(np.abs(s0)) <= tol, f"Position profile must equal [0, 0, 0] at t=0, step(0) returned {s0}"
        s1 = np.asarray(self.step(1))
        assert np.all(np.abs(s1 - 1) <= tol), f"Position profile must equal [1, 1, 1] at t=1, step(1) returned {s1}"

    def step(self, t):
        raise NotImplementedError


class Linear(PosProf):
    """Straight line from [0, 0, 0] to [1, 1, 1]."""

    def __init__(self, n_sample_points=10, **kwargs):
        super().__init__(n_sample_points=n_sample_points, **kwargs)

    def step(self, t):
        return np.array([t, t, t])


class SinCurve(PosProf):
    """Each axis named in ``axes`` (default ["x"]) follows sin(c t pi/2) with c = 4 (cycles - 1) + 1, so that it still
    ends at 1; the others are straight."""

    def __init__(self, axes=None, cycles=None, n_sample_points=1000, **kwargs):
        self.axes = ["x"] if axes is None else axes
        # the caller's list is left as it is (the reference rewrites it in place, so reusing it changes the shape)
        self.cycles = [(cyc - 1) * 4 + 1 for cyc in ([1, 1, 1] if cycles is None else cycles)]
        super().__init__(n_sample_points=n_sample_points, **kwargs)

    def step(self, t):
        out = []
        for i, name in enumerate("xyz"):
            out.append(np.sin(self.cycles[i] * t * np.pi / 2) if name in self.axes else t)
        return np.array(out)


class FromPoints(PosProf):
    """Piecewise-linear profile through the points ``y`` (3, N) or (N, 3) at times ``x`` (N,)."""

    def __init__(self, x, y, n_sample_points=1000, **kwargs):
        y = np.asarray(y, dtype=np.float64)
        if y.shape[0] != 3:
            y = y.T
        self.x = np.asarray(x, dtype=np.float64)
        self.y = y
        super().__init__(n_sample_points=n_sample_points, **kwargs)

    def step(self, t):
        if t == 0:
            return np.zeros(3)
        if t == 1:
            return np.ones(3)
        if t < self.x[0] or t > self.x[-1]:
            raise ValueError(f"t={t} is outside the profile's points [{self.x[0]}, {self.x[-1]}]")
        return np.array([np.interp(t, self.x, self.y[i]) for i in range(3)])


class Ellipse(PosProf):
    """Half ellipse in ``plane`` ("xy" by default) from [0, 0] to [1, 1], bulging sideways by ``horz_stretch`` (to the
    other side when negative); the remaining axis is straight."""

    def __init__(self, horz_stretch, plane="xy", n_sample_points=1000, **kwargs):
        self.indices = {"x": 0, "y": 1, "z": 2}
        self.plane = plane
        self.linear_index = [v for k, v in self.indices.items() if k not in plane][-1]
        self.b = horz_stretch
        g = -np.pi / 4  # rotate the ellipse's chord from the x axis onto [1, 1]
        self.R = np.array([[np.cos(g), -np.sin(g)], [np.sin(g), np.cos(g)]])
        self.mag = 2 * np.sin(-g)
        super().__init__(n_sample_points=n_sample_points, **kwargs)

    def step(self, t):
        y = self.b * np.sqrt(1 - (t - 0.5) ** 2 / 0.5 ** 2)
        xy = np.dot(np.array([t, y]), self.R) * self.mag
        out = np.zeros(3)
        out[self.indices[self.plane[0]]] = xy[0]
        out[self.indices[self.plane[1]]] = xy[1]
        out[self.linear_index] = t
        return out
