"""CPU oracle: host sequence of FusedLAMBAMP.step over the C restatement (lamb_oracle.c).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Follows PyTorch/LanguageModeling/BERT/lamb_amp_opt/fused_lamb/fused_lamb.py:130-260
and schedulers.py:109-136 (PolyWarmUpScheduler).  numpy float32 arrays in, updated in place.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liblamb_oracle.so")
_lib = None


def build(force=False):
    """gcc -O2 -fopenmp -shared oracle/lamb_oracle.c -> oracle/liblamb_oracle.so (no -ffast-math:
    the oracle keeps IEEE division/sqrt)."""
    src = os.path.join(_HERE, "lamb_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-fopenmp", "-fPIC", "-shared", "-o", _SO, src, "-lm"])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_SO)
        fp, i64, f32, dp = ctypes.POINTER(ctypes.c_float), ctypes.c_int64, ctypes.c_float, ctypes.POINTER(ctypes.c_double)
        L.lamb_oracle_sumsq_f32.argtypes = [fp, i64, dp]
        L.lamb_oracle_sumsq_f32.restype = ctypes.c_int
        L.lamb_oracle_stage1_f32.argtypes = [fp, fp, fp, fp, fp, i64, f32, f32, f32, f32, f32, f32,
                                             ctypes.c_int, f32, f32, f32]
        L.lamb_oracle_stage1_f32.restype = ctypes.c_double
        L.lamb_oracle_stage2_f32.argtypes = [fp, fp, i64, f32, f32, f32, f32, ctypes.c_int]
        L.lamb_oracle_stage2_f32.restype = None
        _lib = L
    return _lib


def _p(a):
    assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def sumsq(a):
    out = ctypes.c_double(0.0)
    bad = lib().lamb_oracle_sumsq_f32(_p(a), a.size, ctypes.byref(out))
    return out.value, bool(bad)


def lamb_step(groups, *, scale=1.0, max_grad_norm=1.0, use_nvlamb=False, adam_w_mode=True,
              update_round=None):
    """One FusedLAMBAMP.step.

    groups: list of dicts with keys
        params (list of np.float32 arrays: fp32 params or fp32 masters, updated in place),
        grads  (list of np.float32 arrays: the *scaled* grads, already widened to fp32),
        exp_avg, exp_avg_sq (lists, updated in place),
        lr (float), betas, eps, weight_decay, step (int, updated), bias_correction, grad_averaging.
    scale: GradScaler scale (grads are scale * true grads); inv_scale = float(1/double(scale))
           (fused_lamb.py:153-159).
    update_round: optional f(np.float32 array)->np.float32 array emulating the reference's storage
           of the stage-1 update in the grad dtype (multi_tensor_lamb.cu:160-170 writes it into g).
    Returns dict(found_inf, global_grad_norm, param_norms, update_norms).
    """
    L = lib()
    # found_inf (grad_scaler._check_inf_per_device, fused_lamb.py:148-152) + global norm (:166-191)
    tot, bad = 0.0, False
    for g in groups:
        for a in g["grads"]:
            s, b = sumsq(a)
            tot += s
            bad = bad or b
    gnorm = np.float32(np.sqrt(tot)) if np.isfinite(tot) else np.float32(np.inf)
    out = dict(found_inf=bad or not np.isfinite(gnorm), global_grad_norm=float(gnorm),
               param_norms=[], update_norms=[])
    if out["found_inf"]:
        return out            # noop flag set: every kernel returns early, step not incremented
    inv_scale = np.float32(1.0 / np.float64(np.float32(scale)))
    max_norm = np.float32(max_grad_norm) * np.float32(scale)                  # :165
    clipped = np.float32(gnorm / max_norm) if gnorm > max_norm else np.float32(1.0)   # lamb.cu:77
    for g in groups:
        g["step"] = int(g["step"]) + 1                                        # :201-204
        b1, b2 = (np.float32(x) for x in g["betas"])
        b3 = np.float32(1.0) - b1 if g.get("grad_averaging", True) else np.float32(1.0)
        if g.get("bias_correction", True):
            bc1 = np.float32(1.0) - np.float32(np.power(b1, np.float32(g["step"])))
            bc2 = np.float32(1.0) - np.float32(np.power(b2, np.float32(g["step"])))
        else:
            bc1 = bc2 = np.float32(1.0)
        decay = np.float32(g["weight_decay"])
        for p, gr, m, v in zip(g["params"], g["grads"], g["exp_avg"], g["exp_avg_sq"]):
            psq, _ = sumsq(p)
            pn = np.float32(np.sqrt(psq))
            upd = np.empty_like(p)
            usq = L.lamb_oracle_stage1_f32(_p(gr), _p(p), _p(m), _p(v), _p(upd), p.size,
                                           b1, b2, b3, bc1, bc2, np.float32(g["eps"]),
                                           1 if adam_w_mode else 0, decay, clipped, inv_scale)
            if update_round is not None:
                upd = np.ascontiguousarray(update_round(upd), dtype=np.float32)
                usq, _ = sumsq(upd)
            un = np.float32(np.sqrt(usq))
            L.lamb_oracle_stage2_f32(_p(p), _p(upd), p.size, np.float32(g["lr"]), pn, un, decay,
                                     1 if use_nvlamb else 0)
            out["param_norms"].append(float(pn))
            out["update_norms"].append(float(un))
    return out


def lamb_step_numpy(groups, *, scale=1.0, max_grad_norm=1.0, use_nvlamb=False, adam_w_mode=True):
    """Independent pure-numpy restatement of the same formulas (cross-check of the C file;
    small cases only)."""
    tot = sum(float(np.sum(a.astype(np.float64) ** 2)) for g in groups for a in g["grads"])
    finite = all(np.isfinite(a).all() for g in groups for a in g["grads"])
    gnorm = np.float32(np.sqrt(tot))
    if not finite or not np.isfinite(gnorm):
        return dict(found_inf=True, global_grad_norm=float(gnorm))
    f = np.float32
    inv_scale = f(1.0 / np.float64(f(scale)))
    max_norm = f(max_grad_norm) * f(scale)
    clipped = f(gnorm / max_norm) if gnorm > max_norm else f(1.0)
    for g in groups:
        g["step"] = int(g["step"]) + 1
        b1, b2 = f(g["betas"][0]), f(g["betas"][1])
        b3 = f(1.0) - b1 if g.get("grad_averaging", True) else f(1.0)
        bc1 = f(1.0) - f(np.power(b1, f(g["step"]))) if g.get("bias_correction", True) else f(1.0)
        bc2 = f(1.0) - f(np.power(b2, f(g["step"]))) if g.get("bias_correction", True) else f(1.0)
        decay, eps, lr = f(g["weight_decay"]), f(g["eps"]), f(g["lr"])
        for p, gr, m, v in zip(g["params"], g["grads"], g["exp_avg"], g["exp_avg_sq"]):
            pn = f(np.sqrt(np.sum(p.astype(np.float64) ** 2)))
            sg = (gr * inv_scale) / clipped
            rp = p if decay != 0 else np.zeros_like(p)
            if not adam_w_mode:
                sg = sg + decay * rp
            m[...] = m * b1 + b3 * sg
            v[...] = v * b2 + (f(1.0) - b2) * sg * sg
            upd = (m / bc1) / (np.sqrt(v / bc2) + eps)
            if adam_w_mode:
                upd = upd + decay * rp
            upd = upd.astype(np.float32)
            un = f(np.sqrt(np.sum(upd.astype(np.float64) ** 2)))
            ratio = lr
            if use_nvlamb or decay != 0:
                ratio = lr * (pn / un) if (un != 0 and pn != 0) else lr
            p[...] = p - ratio * upd
    return dict(found_inf=False, global_grad_norm=float(gnorm))


def poly_warmup_lr(step_after, total_steps, warmup, base_lr, degree=0.5):
    """PolyWarmUpScheduler.step/get_lr, schedulers.py:123-136.  `step_after` is
    param_group['step'] (already-taken optimizer steps); last_epoch = step+1 (fp32 math)."""
    f = np.float32
    progress = f(f(step_after + 1) / f(total_steps))
    if progress < f(warmup):
        return float(f(base_lr) * progress / f(warmup))
    return float(f(base_lr) * np.power(f(1.0) - progress, f(degree)))


def adam_step_numpy(groups, *, scale=1.0, max_grad_norm=0.0, clip_eps=1e-6, adam_w_mode=True):
    """CPU oracle for the SQuAD optimizer step: GradientClipper (run_squad.py:716-724: coef = max/(norm + 1e-6), applied when
    < 1) followed by Adam/AdamW as apex.optimizers.FusedAdam is called at run_squad.py:973-975 (bias_correction=False there).
    apex is not vendored in the reference (unpinned): the arithmetic is the published Adam/AdamW update, pinned against
    torch.optim.AdamW in tests/test_lamb_oracle.py.  fp32 element math, double norm."""
    f = np.float32
    tot = sum(float(np.sum(a.astype(np.float64) ** 2)) for g in groups for a in g["grads"])
    finite = all(np.isfinite(a).all() for g in groups for a in g["grads"])
    gnorm = f(np.sqrt(tot))
    if not finite or not np.isfinite(gnorm):
        return dict(found_inf=True, global_grad_norm=float(gnorm))
    inv_scale = f(1.0 / np.float64(f(scale)))
    clip = f(1.0)
    if max_grad_norm > 0:
        max_norm = f(max_grad_norm) * f(scale)
        num = gnorm + f(clip_eps) * f(scale)
        if num > max_norm:
            clip = f(num / max_norm)
    for g in groups:
        g["step"] = int(g["step"]) + 1
        b1, b2 = f(g["betas"][0]), f(g["betas"][1])
        bc1 = f(1.0) - f(np.power(b1, f(g["step"]))) if g.get("bias_correction", True) else f(1.0)
        bc2 = f(1.0) - f(np.power(b2, f(g["step"]))) if g.get("bias_correction", True) else f(1.0)
        wd, eps, lr = f(g["weight_decay"]), f(g["eps"]), f(g["lr"])
        for p, gr, m, v in zip(g["params"], g["grads"], g["exp_avg"], g["exp_avg_sq"]):
            sg = (gr * inv_scale) / clip
            if not adam_w_mode:
                sg = sg + wd * p
            m[...] = m * b1 + (f(1.0) - b1) * sg
            v[...] = v * b2 + (f(1.0) - b2) * sg * sg
            upd = (m / bc1) / (np.sqrt(v / bc2) + eps)
            if adam_w_mode:
                upd = upd + wd * p
            p[...] = p - lr * upd.astype(np.float32)
    return dict(found_inf=False, global_grad_norm=float(gnorm))
