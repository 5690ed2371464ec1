"""float64 references of the FIR stages and the per-VFO gate shared by the sample-by-sample kernel tests
(test_gpu_chain_f64.py, test_gpu_stage1_f64.py)."""
import numpy as np
from scipy.signal import oaconvolve

from util import rel_rms

U = 2.0 ** -24                      # unit round-off of fp32
REF_FLOOR = 2.0 ** -40              # float64 FFT convolution error, relative to sum|h| max|x|: far below any fp32 rounding
EDGE = 64                           # outputs either side of a chunk boundary that count as "edge" in _gate_vfo


def _corr(x, h):
    """z[o] = sum_k h[k] x[o + k] for o = 0 .. len(x) - len(h)  (float64)"""
    if x.size < h.size:
        return np.zeros(0, x.dtype)
    if h.size <= 64 or x.size <= 4 * h.size:
        return np.convolve(x, h[::-1], "valid")
    return oaconvolve(x, h[::-1], "valid")


def _hist(v, k):
    return np.concatenate([np.zeros(k, v.dtype), v])


def _abs_parts(x):
    return np.abs(x.real) + (np.abs(x.imag) if np.iscomplexobj(x) else 0.0)


def fir_f64(x, e, h, D=1):
    """FIR / DecimatingFIR from zero history: y[m] = sum_k h[k] xh[m D + k], xh = [T-1 zeros | x].
    x: float64 input, e: per-sample bound of x's error (None = exact fp32 input).  Returns (y, bound of y)."""
    h = np.asarray(h, np.float64)
    T = h.size
    y = _corr(_hist(x, T - 1), h)[::D]
    a = _abs_parts(x) + (2.0 * e if e is not None else 0.0)
    ah = np.abs(h)
    b = (T + 2) * U * _corr(_hist(a, T - 1), ah)[::D]
    if e is not None:
        b = b + _corr(_hist(e, T - 1), ah)[::D]
    return y, b + REF_FLOOR * ah.sum() * (float(a.max()) if a.size else 0.0)


def _gate_vfo(parts_gpu, parts_ref):
    """count, rel_rms, fitted complex gain and edge-against-interior for one VFO"""
    assert [p.size for p in parts_gpu] == [p.size for p in parts_ref]
    y = np.concatenate(parts_gpu).astype(np.complex128)
    yo = np.concatenate(parts_ref).astype(np.complex128)
    e_rms = rel_rms(y, yo)
    g = np.vdot(yo, y) / np.vdot(yo, yo)
    e = np.abs(y - yo) / np.sqrt(np.mean(np.abs(yo) ** 2))
    edge = np.zeros(y.size, bool)
    for b in np.cumsum([0] + [p.size for p in parts_ref[:-1]]):
        edge[max(0, b - EDGE): b + EDGE] = True
    assert edge.any() and (~edge).sum() >= 1000
    p999 = float(np.percentile(e[~edge], 99.9))
    ratio = float(e[edge].max() / p999) if p999 > 0 else (0.0 if e[edge].max() == 0 else np.inf)
    return {"rel_rms": e_rms, "gain_re": float(g.real), "gain_im": float(g.imag), "abs_g_minus_1": float(abs(g - 1)),
            "edge_over_p999": ratio, "outputs": int(y.size)}
