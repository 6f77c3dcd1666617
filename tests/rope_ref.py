"""A numpy statement of the rope shift (b200kv_rope_shift): the keys' rotary channels turned by shift·inv_freq[j], the
angle and the rotation in float64.  Pairs: neox (d, d + rotary_dim/2), gptj (2d, 2d + 1); channels [offset, offset +
rotary_dim) of the last axis; everything else as it is.  Plus the tolerance the kernel is held to."""
import numpy as np


def angles(shift, inv_freq):
    """[..., half] angles: float64(shift) * float64(float32 inv_freq), shift a scalar or an array of per-row shifts"""
    s = np.asarray(shift, dtype=np.float64)
    return s[..., None] * np.asarray(inv_freq, dtype=np.float32).astype(np.float64)


def _pairs(rotary_dim, style, offset):
    half = rotary_dim // 2
    if style == "neox":
        return np.arange(offset, offset + half), np.arange(offset + half, offset + rotary_dim)
    if style == "gptj":
        return np.arange(offset, offset + rotary_dim, 2), np.arange(offset + 1, offset + rotary_dim, 2)
    raise ValueError(style)


def rotate(k, shift, inv_freq, rotary_dim, style="neox", offset=0):
    """k: float64 [n, ..., D]; shift: a scalar or [n] per-row shifts.  Returns the rotated copy (float64)."""
    k = np.asarray(k, dtype=np.float64)
    a, b = _pairs(rotary_dim, style, offset)
    ang = angles(shift, inv_freq)                       # [half] or [n, half]
    if ang.ndim == 2:
        ang = ang.reshape(ang.shape[:1] + (1,) * (k.ndim - 2) + ang.shape[1:])
    c, s = np.cos(ang), np.sin(ang)
    x, y = k[..., a], k[..., b]
    out = k.copy()
    out[..., a] = x * c - y * s
    out[..., b] = y * c + x * s
    return out


def rotate_complex(k, shift, inv_freq, rotary_dim, style="neox", offset=0):
    """the same rotation as the product of (x + iy) with exp(i·angle)"""
    k = np.asarray(k, dtype=np.float64)
    a, b = _pairs(rotary_dim, style, offset)
    ang = angles(shift, inv_freq)
    if ang.ndim == 2:
        ang = ang.reshape(ang.shape[:1] + (1,) * (k.ndim - 2) + ang.shape[1:])
    z = (k[..., a] + 1j * k[..., b]) * np.exp(1j * ang)
    out = k.copy()
    out[..., a], out[..., b] = z.real, z.imag
    return out


def partner(rotary_dim, style, offset, D):
    """[D] channel index of each channel's rotation partner (itself outside the rotary range)"""
    p = np.arange(D)
    a, b = _pairs(rotary_dim, style, offset)
    p[a], p[b] = b, a
    return p


# significand bits after the leading one, and the smallest ulp (of the subnormals)
_FMT = {"bfloat16": (7, 2.0 ** -133), "float16": (10, 2.0 ** -24)}


def ulp(v, dtype_name):
    """the ulp of |v| in the dtype (float64 arrays in, float64 out)"""
    m, tiny = _FMT[dtype_name]
    v = np.abs(np.asarray(v, dtype=np.float64))
    e = np.floor(np.log2(np.where(v > 0, v, 1.0)))
    return np.maximum(np.where(v > 0, 2.0 ** (e - m), tiny), tiny)


def tolerance(ref_rounded, got, x, y, dtype_name):
    """what the kernel may differ from the float64 statement rounded to the dtype: one ulp (of either value), plus the
    fp32 error of the rotation itself, at most 2^-21 (|x| + |y|) -- visible only when the pair nearly cancels, where
    the result's ulp is far below its operands' (x, y: the pair's inputs)"""
    return np.maximum(ulp(ref_rounded, dtype_name), ulp(got, dtype_name)) + 2.0 ** -21 * (np.abs(x) + np.abs(y))
