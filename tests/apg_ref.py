"""Float64 model of adaptive projected guidance (APG; Sadat, Hilliges, Weber, ICLR 2025, arXiv:2410.02416) as
include/ivid_b200.h defines it, for one step and for a chain of steps with momentum, and the fp32 error bound of the device's
arithmetic.  Arrays are [N, ...]: every norm and inner product runs over one sample's elements."""
import numpy as np

TINY = np.finfo(np.float64).tiny
EPS32 = float(np.finfo(np.float32).eps)
SUBNORMAL32 = float(np.finfo(np.float32).smallest_subnormal)


def _flat(a):
    a = np.asarray(a, dtype=np.float64)
    return a.reshape(a.shape[0], -1)


def scalars(dc, m, s, eta, r):
    """c and k of every sample: c = min(1, r / |m|) (1 for r = 0 or m = 0), k = (1 - eta) <m, D_c> / max(|D_c|^2, tiny)."""
    dc, m = _flat(dc), _flat(m)
    nm = np.sqrt((m * m).sum(axis=1))
    c = np.ones_like(nm)
    if r > 0:
        live = nm > 0
        c[live] = np.minimum(1.0, r / nm[live])
    k = (1.0 - eta) * (m * dc).sum(axis=1) / np.maximum((dc * dc).sum(axis=1), TINY)
    return c, k


def apg64(dc, du, s, eta=0.0, r=0.0, beta=0.0, m_prev=None, pag=None):
    """One guided step: (D, m).  dc / du are D_c / D_u, m_prev the momentum state (None: zero history), pag the PAG term
    w (D_c - D_p) added to D (None: no PAG)."""
    shape = np.shape(dc)
    dc, du = _flat(dc), _flat(du)
    m = dc - du
    if m_prev is not None and beta != 0.0:
        m = m + beta * _flat(m_prev)
    c, k = scalars(dc, m, s, eta, r)
    d = dc + (s * c)[:, None] * (m - k[:, None] * dc)
    if pag is not None:
        d = d + _flat(pag)
    return d.reshape(shape), m.reshape(shape)


def chain64(dcs, dus, s, eta=0.0, r=0.0, beta=0.0):
    """A run of guided steps from zero history: the list of D and the final m."""
    m, out = None, []
    for dc, du in zip(dcs, dus):
        d, m = apg64(dc, du, s, eta, r, beta, m)
        out.append(d)
    return out, m


def bound32(dc, du, s, eta=0.0, r=0.0, beta=0.0, m_prev=None):
    """Per-element bound on |D_device - D_model| for fp32 inputs: the device rounds D_c - D_u (1 op), the momentum (2), the
    scalars s c and s c k (one rounding each, and c itself), and D_c + (a m - b D_c) (4).  Each rounding contributes at most
    one unit of the magnitude it acts on, so the bound is a small multiple of eps32 times the terms' magnitudes.  One term is
    global: the rounding of m moves <m, D_c> by up to eps |m| |D_c|, so k by eps |m| / |D_c|, which reaches every element
    as s c (eps |m| / |D_c|) |D_c[i]|."""
    shape = np.shape(dc)
    dcf, duf = _flat(dc), _flat(du)
    mp = np.zeros_like(dcf) if m_prev is None else _flat(m_prev)
    m = dcf - duf + beta * mp
    c, k = scalars(dcf, m, s, eta, r)
    a, b = np.abs(s * c)[:, None], np.abs(s * c * k)[:, None]
    mag_m = m_bound_mag(dcf, duf, beta, mp)
    ndc = np.sqrt((dcf * dcf).sum(axis=1))
    proj = np.zeros_like(ndc)                  # D_c = 0: k = 0 exactly
    live = ndc > 0
    proj[live] = (1.0 - eta) * np.sqrt((mag_m[live] ** 2).sum(axis=1)) / ndc[live]
    rel = 8 * EPS32 * (np.abs(dcf) + a * mag_m + b * np.abs(dcf) + a * proj[:, None] * np.abs(dcf))
    # below 2^-126 a rounding errs by up to half the subnormal spacing 2^-149, whatever the magnitude
    return (rel + 8 * (1 + a + b) * SUBNORMAL32).reshape(shape)


def m_bound_mag(dc, du, beta, m_prev):
    """The magnitude the rounding of m = D_c - D_u + beta m_prev acts on, per element (D_c, D_u themselves carry one
    rounding of their own size when they come from a step): |D_c| + |D_u| + |beta m_prev|."""
    return np.abs(dc) + np.abs(du) + abs(beta) * np.abs(m_prev)
