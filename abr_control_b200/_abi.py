"""ctypes mirror of include/abrb.h (struct layouts and constants only; no library loading here)."""
import ctypes as C
import math
import json
import os

MAX_JOINTS = 7
MAX_NULL = 4
MAX_OBSTACLES = 16

OK, EINVAL, EFRAME, ESHAPE, EUNSUP, ECUDA, ENOMEM = 0, -1, -2, -3, -4, -5, -6
NULL_DAMPING, NULL_RESTING, NULL_AVOID, NULL_JOINT_LIMITS = 1, 2, 3, 4


class ChainDesc(C.Structure):
    _fields_ = [
        ("n_joints", C.c_int32),
        ("n_links", C.c_int32),
        ("L0", C.c_double * 12),
        ("A", (C.c_double * 12) * MAX_JOINTS),
        ("B", (C.c_double * 12) * MAX_JOINTS),
        ("E", C.c_double * 12),
        ("link_inertia", (C.c_double * 6) * (MAX_JOINTS + 1)),
        ("gravity", C.c_double * 6),
    ]


class RbdOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("Tx", "T", "R", "T_inv", "quat", "J", "dJ", "M", "g", "C")]


class NullParams(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("n_obstacles", C.c_int32),
        ("kp", C.c_double),
        ("kv", C.c_double),
        ("rest_angles", C.c_double * MAX_JOINTS),
        ("rest_mask", C.c_int32 * MAX_JOINTS),
        ("_pad", C.c_int32),
        ("threshold", C.c_double),
        ("gain", C.c_double),
        ("maximum", C.c_double),
        ("obstacles", (C.c_double * 4) * MAX_OBSTACLES),
        ("limit_min", C.c_double * MAX_JOINTS),
        ("limit_max", C.c_double * MAX_JOINTS),
        ("limit_torque", C.c_double * MAX_JOINTS),
        ("limit_cross_zero", C.c_int32 * MAX_JOINTS),
        ("limit_gradient", C.c_int32 * MAX_JOINTS),
    ]


# include/abrb.h abrb_path_params / abrb_path_rec (the batched path planner)
PATH_MAX_POINTS = 4096
VEL_GAUSSIAN, VEL_LINEAR = 0, 1


class PathParams(C.Structure):
    _fields_ = [
        ("vel_kind", C.c_int32),
        ("n_points", C.c_int32),
        ("dt", C.c_double),
        ("acceleration", C.c_double),
        ("n_sigma", C.c_double),
        ("axes", C.c_int32 * 4),
    ]


class PathRec(C.Structure):
    _fields_ = [("max_v", C.c_double), ("n_start", C.c_int32), ("n_const", C.c_int32), ("n_end", C.c_int32),
                ("flags", C.c_int32)]


class OscParams(C.Structure):
    _fields_ = [
        ("kp", C.c_double),
        ("ko", C.c_double),
        ("kv", C.c_double),
        ("ki", C.c_double),
        ("vmax", C.c_double * 2),
        ("mx_threshold", C.c_double),
        ("use_vmax", C.c_int32),
        ("ctrlr_dof", C.c_int32 * 6),
        ("use_g", C.c_int32),
        ("use_C", C.c_int32),
        ("orientation_algorithm", C.c_int32),
        ("n_null", C.c_int32),
        ("_pad", C.c_int32),
        ("null", NullParams * MAX_NULL),
    ]


DATA_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "arms", "data")


def load_arm_json(arm):
    with open(os.path.join(DATA_DIR, f"{arm}.json")) as fh:
        return json.load(fh)


def chain_desc_from_dict(d):
    """Flat chain descriptor (dict as stored in arms/data/*.json) -> ChainDesc."""
    n = int(d["n_joints"])
    if not 1 <= n <= MAX_JOINTS:
        raise ValueError(f"n_joints={n} outside [1, {MAX_JOINTS}]")
    cd = ChainDesc()
    cd.n_joints = n
    cd.n_links = int(d["n_links"])

    def put(dst, m34):
        flat = [float(v) for row in m34 for v in row]
        assert len(flat) == 12
        for i, v in enumerate(flat):
            dst[i] = v

    put(cd.L0, d["L0"])
    put(cd.E, d["E"])
    for i in range(n):
        put(cd.A[i], d["A"][i])
        put(cd.B[i], d["B"][i])
    for l in range(cd.n_links):
        for c in range(6):
            cd.link_inertia[l][c] = float(d["link_inertia"][l][c])
    for c in range(6):
        cd.gravity[c] = float(d["gravity"][c])
    return cd


def null_params(kind, n_joints, kv=None, kp=1.0, rest_angles=None, obstacles=None, threshold=0.2, gain=1.0,
                maximum=500.0, min_joint_angles=None, max_joint_angles=None, max_torque=None, cross_zero=None,
                gradient=None):
    """Build a NullParams with the reference's constructor defaults
    (damping.py:15-19, joint.py:29-36 + resting_config.py:18-23, avoid_obstacles.py:25-36,
    avoid_joint_limits.py:36-86)."""
    z = NullParams()
    if kind == "Damping":
        z.kind = NULL_DAMPING
        z.kv = float(kv)
    elif kind == "RestingConfig":
        z.kind = NULL_RESTING
        z.kp = float(kp)
        z.kv = float(kp) ** 0.5 if kv is None else float(kv)
        if len(rest_angles) != n_joints:
            raise ValueError("rest_angles must have one entry per joint")
        for k, v in enumerate(rest_angles):
            z.rest_mask[k] = 0 if v is None else 1
            z.rest_angles[k] = 0.0 if v is None else float(v)
    elif kind == "AvoidObstacles":
        z.kind = NULL_AVOID
        obstacles = [] if obstacles is None else list(obstacles)
        if len(obstacles) > MAX_OBSTACLES:
            raise ValueError(f"at most {MAX_OBSTACLES} obstacles")
        z.n_obstacles = len(obstacles)
        for i, ob in enumerate(obstacles):
            for c in range(4):
                z.obstacles[i][c] = float(ob[c])
        z.threshold, z.gain, z.maximum = float(threshold), float(gain), float(maximum)
    elif kind == "AvoidJointLimits":
        z.kind = NULL_JOINT_LIMITS
        if len(min_joint_angles) != n_joints or len(max_joint_angles) != n_joints:
            raise Exception("joint angles vector incorrect size")  # avoid_joint_limits.py:68-72
        nan = float("nan")
        # the constructor shifts the limits to the -pi..pi range (:46-51) and swaps them where the working range
        # crosses zero (:62-66); None (or NaN) = no limit on that side
        lo = [nan if v is None else float(v) - math.pi for v in min_joint_angles]
        hi = [nan if v is None else float(v) - math.pi for v in max_joint_angles]
        cz = [False] * n_joints if cross_zero is None else [bool(v) for v in cross_zero]
        gr = [False] * n_joints if gradient is None else [bool(v) for v in gradient]
        tq = [1.0] * n_joints if max_torque is None else [float(v) for v in max_torque]
        for k in range(n_joints):
            z.limit_min[k], z.limit_max[k] = (hi[k], lo[k]) if cz[k] else (lo[k], hi[k])
            z.limit_torque[k] = tq[k]
            z.limit_cross_zero[k], z.limit_gradient[k] = int(cz[k]), int(gr[k])
    else:
        raise ValueError(f"unknown secondary controller {kind}")
    return z


def osc_params(n_joints, kp=1, ko=None, kv=None, ki=0, vmax=None, ctrlr_dof=None, null=None, use_g=True,
               use_C=False, orientation_algorithm=0, mx_threshold=1e-3):
    """OscParams with the reference's defaults resolved (controllers/osc.py:53-118)."""
    p = OscParams()
    p.kp = float(kp)
    p.ko = float(kp if ko is None else ko)
    p.kv = float((p.kp + p.ko) ** 0.5 if kv is None else kv)
    p.ki = float(ki)
    p.use_vmax = 0 if vmax is None else 1
    if vmax is not None:
        p.vmax[0], p.vmax[1] = float(vmax[0]), float(vmax[1])
    p.mx_threshold = float(mx_threshold)
    dof = [True, True, True, False, False, False] if ctrlr_dof is None else list(ctrlr_dof)
    if len(dof) != 6:
        raise ValueError("ctrlr_dof must have 6 entries")
    for r in range(6):
        p.ctrlr_dof[r] = 1 if dof[r] else 0
    p.use_g, p.use_C = int(bool(use_g)), int(bool(use_C))
    p.orientation_algorithm = int(orientation_algorithm)
    null = [] if null is None else list(null)
    if len(null) > MAX_NULL:
        raise ValueError(f"at most {MAX_NULL} null controllers")
    p.n_null = len(null)
    for i, z in enumerate(null):
        p.null[i] = z
    return p
