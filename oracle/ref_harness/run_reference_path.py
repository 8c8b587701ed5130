#!/usr/bin/env python
"""TEST INFRASTRUCTURE (development container only): run the reference's PathPlanner and write
tests/golden/path_planner.npz.

    PYTHONPATH=/root/reference python -W ignore oracle/ref_harness/run_reference_path.py

The reference is run unmodified; its modules import matplotlib for optional plots, which the image does not have, so
the harness registers the same empty stand-ins as run_reference.py (the plotting branches are never taken).  The
fixture holds, per case, the inputs, the profile's sampled table and the path the reference returned (data only).
Case i is stored under keys "c<i>_*"; "meta" is a JSON list with each case's profile and planner specification.
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))

for mod in ("matplotlib", "matplotlib.pyplot", "mpl_toolkits", "mpl_toolkits.mplot3d"):
    sys.modules.setdefault(mod, types.ModuleType(mod))
sys.modules["mpl_toolkits.mplot3d"].axes3d = None

from abr_control.controllers.path_planners import path_planner as pp_mod  # noqa: E402
from abr_control.controllers.path_planners import position_profiles as pos  # noqa: E402
from abr_control.controllers.path_planners import velocity_profiles as vel  # noqa: E402

FP_X = [0.0, 0.3, 0.7, 1.0]
FP_Y = [[0.0, 0.0, 0.0], [0.5, 0.1, 0.2], [0.6, 0.9, 0.5], [1.0, 1.0, 1.0]]

# (position profile, velocity profile, planner kwargs, generate_path kwargs)
CASES = [
    (("Linear", {}), ("Gaussian", {"dt": 0.002, "acceleration": 5}), "rxyz",
     dict(start=[0.1, 0.2, 0.3], target=[0.5, -0.1, 0.6], max_velocity=1.0, so=[0.1, 0.2, 0.3], to=[-0.4, 0.5, 1.2])),
    (("Linear", {}), ("Linear", {"dt": 0.002, "acceleration": 5}), "rxyz",
     dict(start=[0.1, 0.2, 0.3], target=[0.5, -0.1, 0.6], max_velocity=1.0, so=[0.1, 0.2, 0.3], to=[-0.4, 0.5, 1.2])),
    (("SinCurve", {"axes": ["x", "z"], "cycles": [1, 1, 2]}), ("Gaussian", {"dt": 0.002, "acceleration": 4}), "sxyz",
     dict(start=[-0.2, 0.4, 0.5], target=[0.3, 0.1, 0.2], max_velocity=0.8, so=[0.3, -0.2, 0.1], to=[1.0, 0.4, -0.7])),
    (("Ellipse", {"horz_stretch": 0.5}), ("Gaussian", {"dt": 0.002, "acceleration": 5}), "rxyz",
     dict(start=[0.0, 0.3, 0.4], target=[0.4, 0.0, 0.6], max_velocity=1.0, so=[0.0, 0.0, 0.0], to=[0.5, -0.5, 2.5])),
    (("Ellipse", {"horz_stretch": -0.8, "plane": "yz"}), ("Linear", {"dt": 0.002, "acceleration": 3}), "rzxz",
     dict(start=[0.2, -0.3, 0.4], target=[-0.2, 0.2, 0.7], max_velocity=0.9, so=[0.2, 0.7, -0.3], to=[-1.0, 1.2, 0.4])),
    (("FromPoints", {"x": FP_X, "y": FP_Y, "n_sample_points": 200}), ("Gaussian", {"dt": 0.002, "acceleration": 5}),
     "rxyz", dict(start=[0.3, 0.3, 0.3], target=[0.0, 0.5, 0.9], max_velocity=1.0, so=[0.1, 0.1, 0.1],
                  to=[0.2, -0.3, 0.4])),
    # start / target velocities: non-zero, equal, and equal to max_velocity (the [v dt] ramps)
    (("Linear", {}), ("Gaussian", {"dt": 0.002, "acceleration": 5}), "rxyz",
     dict(start=[0.0, 0.0, 0.0], target=[0.6, 0.2, -0.3], max_velocity=1.0, start_velocity=0.3, target_velocity=0.5)),
    (("Linear", {}), ("Linear", {"dt": 0.002, "acceleration": 5}), "rxyz",
     dict(start=[0.0, 0.0, 0.0], target=[0.61, 0.2, -0.3], max_velocity=1.0, start_velocity=0.4, target_velocity=0.4)),
    (("Linear", {}), ("Gaussian", {"dt": 0.002, "acceleration": 5}), "rxyz",
     dict(start=[0.1, 0.0, 0.0], target=[0.5, 0.6, -0.3], max_velocity=0.8, start_velocity=0.8, target_velocity=0.0,
          so=[0.5, 0.1, 0.2], to=[0.1, 0.2, 0.3])),
    (("SinCurve", {}), ("Linear", {"dt": 0.002, "acceleration": 5}), "rxyz",
     dict(start=[0.1, 0.0, 0.0], target=[0.5, 0.6, -0.3], max_velocity=0.8, start_velocity=0.0, target_velocity=0.8)),
    (("Linear", {}), ("Gaussian", {"dt": 0.002, "acceleration": 5}), "rxyz",
     dict(start=[0.1, 0.0, 0.0], target=[0.5, 0.6, -0.3], max_velocity=0.7, start_velocity=0.7, target_velocity=0.7)),
    # short reaches: the max_v search steps down
    (("Linear", {}), ("Gaussian", {"dt": 0.002, "acceleration": 2}), "rxyz",
     dict(start=[0.0, 0.0, 0.0], target=[0.05, 0.03, 0.02], max_velocity=1.0, so=[0.0, 0.3, 0.0], to=[0.2, 0.0, 0.1])),
    (("Ellipse", {"horz_stretch": 0.3}), ("Linear", {"dt": 0.002, "acceleration": 1}), "sxyx",
     dict(start=[0.0, 0.2, 0.0], target=[0.1, 0.1, 0.05], max_velocity=1.0, so=[0.3, 1.2, -0.4], to=[-0.2, 0.6, 0.9])),
    (("SinCurve", {"axes": ["y"]}), ("Gaussian", {"dt": 0.001, "acceleration": 3}), "ryzy",
     dict(start=[0.2, 0.2, 0.2], target=[0.3, 0.25, 0.05], max_velocity=1.5, start_velocity=0.2,
          so=[2.5, 0.4, -2.8], to=[-2.9, 0.8, 2.6])),
    # a reach through the opposite quadrant (rotation of the shape by more than 90 degrees), and the default n_sigma
    (("Ellipse", {"horz_stretch": 0.4, "plane": "xz"}), ("Gaussian", {"dt": 0.002, "acceleration": 5, "n_sigma": 2}),
     "szyx", dict(start=[0.4, 0.4, 0.4], target=[0.1, 0.0, 0.2], max_velocity=1.2, so=[3.0, 0.2, -3.0],
                  to=[-3.0, -0.2, 3.0])),
]


def make_pos(name, kw):
    kw = dict(kw)
    if name == "FromPoints":
        kw["x"] = np.array(kw["x"])
        kw["y"] = np.array(kw["y"]).T
    if name == "SinCurve":
        kw = {k: list(v) if isinstance(v, list) else v for k, v in kw.items()}
    return getattr(pos, name)(**kw)


def main():
    out, meta = {}, []
    for i, ((pname, pkw), (vname, vkw), axes, g) in enumerate(CASES):
        prof = make_pos(pname, pkw)
        vp = getattr(vel, vname)(**vkw)
        planner = pp_mod.PathPlanner(prof, vp, axes=axes)
        table = np.array([prof.step(t) for t in np.linspace(0, 1, prof.n_sample_points)], dtype=np.float64)
        start, target = np.array(g["start"], dtype=np.float64), np.array(g["target"], dtype=np.float64)
        kw = dict(max_velocity=g["max_velocity"], start_velocity=g.get("start_velocity", 0),
                  target_velocity=g.get("target_velocity", 0))
        if "so" in g:
            kw.update(start_orientation=np.array(g["so"], dtype=np.float64),
                      target_orientation=np.array(g["to"], dtype=np.float64))
        path = planner.generate_path(start, target, plot=False, **kw)
        out[f"c{i}_table"] = table
        out[f"c{i}_start"], out[f"c{i}_target"] = start, target
        out[f"c{i}_speeds"] = np.array([kw["max_velocity"], kw["start_velocity"], kw["target_velocity"]], dtype=float)
        if "so" in g:
            out[f"c{i}_so"], out[f"c{i}_to"] = kw["start_orientation"], kw["target_orientation"]
        out[f"c{i}_path"] = np.asarray(path, dtype=np.float64)
        meta.append(dict(pos=[pname, pkw], vel=[vname, vkw], axes=axes, orient="so" in g))
        print(f"case {i}: {pname}/{vname} {axes} S={len(path)}", flush=True)
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "path_planner.npz"), **out)


if __name__ == "__main__":
    main()
