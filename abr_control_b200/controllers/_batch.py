"""Shared input/output plumbing for the batched controllers (host NumPy buffers or CUDA torch tensors)."""
import numpy as np

try:
    import torch
except Exception:  # pragma: no cover
    torch = None


def is_torch(x):
    return torch is not None and isinstance(x, torch.Tensor)


def prep_state(rc, q, dq):
    """-> (q2, dq2, single, kind, f32) with q2/dq2 contiguous (B, n)."""
    qa, single, kind = rc._prep(q, np.float64 if (np.ndim(q) == 1 and not is_torch(q)) else None)
    dqa, _, kind2 = rc._prep(dq, qa.dtype if kind == "numpy" else None)
    if kind != kind2 or qa.shape != dqa.shape or (kind == "torch" and qa.dtype != dqa.dtype):
        raise ValueError("q and dq must have the same type, dtype and shape")
    f32 = (qa.dtype == torch.float32) if kind == "torch" else (qa.dtype == np.float32)
    return qa, dqa, single, kind, f32


def prep_rows(x, like, kind, width, what):
    """(width,) -> broadcast row (stride 0); (B, width) -> per-state rows (stride width)."""
    B = like.shape[0]
    if kind == "torch":
        t = x if is_torch(x) else torch.as_tensor(np.asarray(x, dtype=np.float64), device=like.device)
        t = t.to(device=like.device, dtype=like.dtype)
        if t.dim() == 1 and t.shape[0] == width:
            return t.contiguous(), 0
        if t.dim() == 2 and t.shape == (B, width):
            return t.contiguous(), width
    else:
        a = np.asarray(x.detach().cpu() if is_torch(x) else x, dtype=like.dtype)
        if a.ndim == 1 and a.shape[0] == width:
            return np.ascontiguousarray(a), 0
        if a.ndim == 2 and a.shape == (B, width):
            return np.ascontiguousarray(a), width
    raise ValueError(f"{what} must have shape ({width},) or ({B}, {width})")


def ptr(a):
    if a is None:
        return None
    return a.data_ptr() if is_torch(a) else a.ctypes.data


def ctrl_rollout(rc, fns, gains, q, dq, rows, width, dt, ref_frame, offset, record, effort_weight, what):
    """Shared plumbing of ``Joint.rollout_path`` and ``Sliding.rollout_path`` (abrb_joint_rollout_path_*,
    abrb_sliding_rollout_path_*).  ``fns``: (f64, f32) entry point names; ``gains``: the controller's leading scalar
    arguments; ``rows``: [(array or None, name)] in the entry point's order, the first being the path, each ``(S,
    width)`` or ``(S, B, width)``.  -> ``(q_final, dq_final, traj, cost)`` in the input's form."""
    import ctypes as C

    from .. import _lib

    qa, dqa, single, kind, f32 = prep_state(rc, q, dq)
    if kind == "numpy":
        dev = torch.device("cuda", torch.cuda.current_device())
        qa, dqa = torch.as_tensor(qa).to(dev), torch.as_tensor(dqa).to(dev)
    else:
        qa, dqa = qa.clone(), dqa.clone()
    B, n = qa.shape

    def prep(x, name):
        t = x if is_torch(x) else torch.as_tensor(np.asarray(x, dtype=np.float64))
        t = t.to(device=qa.device, dtype=qa.dtype).contiguous()
        if t.dim() == 2 and t.shape[1] == width:
            return t, 0
        if t.dim() == 3 and t.shape[1:] == (B, width):
            return t, width
        raise ValueError(f"{name} must have shape (S, {width}) or (S, {B}, {width})")

    args, steps = [], None
    for x, name in rows:
        if x is None:
            args += [None, 0]
            continue
        t, stride = prep(x, name)
        if steps is None:
            steps = t.shape[0]
        elif t.shape[0] != steps:
            raise ValueError(f"{name} has {t.shape[0]} steps, {rows[0][1]} has {steps}")
        args += [t, stride]
    fid = rc.frame_id(ref_frame)
    xo = None
    if offset is not None and not np.allclose(np.asarray(offset, dtype=float), 0):
        xo = (C.c_double * 3)(*[float(v) for v in np.asarray(offset, dtype=float).reshape(3)])
    for k in record:
        if k not in ("q", "dq", "u", "x"):
            raise ValueError(f"{what} can record 'q', 'dq', 'u' and 'x', not {k!r}")
    traj = {k: torch.empty((steps, B, 3 if k == "x" else n), dtype=qa.dtype, device=qa.device) for k in record}
    cost = torch.empty((B,), dtype=qa.dtype, device=qa.device)
    fn = getattr(_lib.lib(), fns[1] if f32 else fns[0])
    with torch.cuda.device(qa.device):
        _lib.check(fn(rc.handle, *gains, fid, xo, qa.data_ptr(), dqa.data_ptr(),
                      *[ptr(a) if i % 2 == 0 else a for i, a in enumerate(args)], int(steps), float(dt),
                      float(effort_weight), ptr(traj.get("q")), ptr(traj.get("dq")), ptr(traj.get("u")),
                      ptr(traj.get("x")), cost.data_ptr(), B, torch.cuda.current_stream(qa.device).cuda_stream))
    if kind == "numpy":
        qa, dqa, cost = qa.cpu().numpy(), dqa.cpu().numpy(), cost.cpu().numpy()
        traj = {k: v.cpu().numpy() for k, v in traj.items()}
    if single:
        return qa[0], dqa[0], {k: v[:, 0] for k, v in traj.items()}, cost[0]
    return qa, dqa, traj, cost


def host_out(shape, dtype):
    """NumPy result buffer for the host-pointer entry points.  From 64 KiB up it is page-locked (torch's caching host
    allocator: cheap after the first call, returned to the cache when the array is dropped) so that the library's
    device->host copy is a plain DMA instead of a staged copy through the driver's bounce buffer."""
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    if nbytes >= (1 << 16):
        import torch

        t = torch.empty(tuple(int(s) for s in shape), dtype=torch.float32 if np.dtype(dtype) == np.float32 else torch.float64,
                        pin_memory=True)
        return t.numpy()  # keeps `t` alive
    return np.empty(shape, dtype=dtype)

