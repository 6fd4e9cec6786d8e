"""Float64 models of the restoration filters, the colour stage and upsampling, and exact integer models of inverse RCT and
Squeeze, written from the reference's Rust sources (crates/jxl-render/src/filter/{gabor,epf}.rs and
impls/generic/{gabor,epf}.rs, crates/jxl-render/src/util.rs, crates/jxl-render/src/features/upsampling.rs,
crates/jxl-color/src/xyb.rs, crates/jxl-modular/src/transform/{rct,squeeze}.rs) rather than from the oracle, so that a
misreading shared by the oracle and the kernels shows up as a disagreement with these.

Each float model returns (value, bound): `bound` is a per-sample limit on |f32 evaluation - float64 value| derived from the
operation count and the operand magnitudes (unit roundoff u = 2^-24, gamma(n) = n u / (1 - n u), Higham's notation),
plus the propagated limit `err_in` of the inputs where a stage takes one (chained EPF steps, the colour stage). A kernel
or oracle output outside the bound is wrong.
"""
import numpy as np

U = 2.0 ** -24
F32 = np.float32


def gamma(n):
    return n * U / (1.0 - n * U)


def mirror(i, n):
    """util.rs:376-386: reflect with the edge sample repeated, as often as needed (period 2n)."""
    m = np.mod(i, 2 * n)
    return np.where(m >= n, 2 * n - 1 - m, m)


def _shifter(a, reach):
    """shift(dx, dy)[y, x] = a[mirror(y + dy), mirror(x + dx)] for |dx|, |dy| <= reach."""
    h, w = a.shape
    ys = mirror(np.arange(-reach, h + reach), h)
    xs = mirror(np.arange(-reach, w + reach), w)
    p = a[np.ix_(ys, xs)]
    return lambda dx, dy: p[reach + dy: reach + dy + h, reach + dx: reach + dx + w]


# ---- Gaborish (gabor.rs) ----------------------------------------------------------------------------------------------

GAB_DEFAULT = (float(F32(0.115169525)), float(F32(0.061248592)))


def gaborish(x, w0, w1, swap_weights=False):
    """One channel. A 3x3 kernel (centre 1, sides w0, corners w1) normalised by 1 / (1 + 4 w0 + 4 w1) over mirrored
    samples - except in a one-row image with at least two columns, where gabor_row_edge's single-row branch weighs the
    centre with 1 + 2 + w0 instead of 1 + 2 w0 (impls/generic/gabor.rs:65-66); the reference decides, so the model
    follows it. `swap_weights` is a planted error for the negative controls."""
    x = np.asarray(x, dtype=np.float64)
    h, w = x.shape
    if swap_weights:
        w0, w1 = w1, w0
    gw = 1.0 / (1.0 + 4.0 * w0 + 4.0 * w1)
    s = _shifter(x, 1)
    a = _shifter(np.abs(x), 1)
    if h == 1 and w == 1:
        out, mag = x.copy(), np.zeros_like(x)
    elif h == 1:
        mw0, mw1 = 3.0 + w0, w0 + 2.0 * w1
        out = (x * mw0 + (s(-1, 0) + s(1, 0)) * mw1) * gw
        mag = (np.abs(x) * mw0 + (a(-1, 0) + a(1, 0)) * mw1) * gw
    else:
        side = s(0, -1) + s(-1, 0) + s(1, 0) + s(0, 1)
        diag = s(-1, -1) + s(1, -1) + s(-1, 1) + s(1, 1)
        out = (x + side * w0 + diag * w1) * gw
        mag = (np.abs(x) + (a(0, -1) + a(-1, 0) + a(1, 0) + a(0, 1)) * w0 +
               (a(-1, -1) + a(1, -1) + a(-1, 1) + a(1, 1)) * w1) * gw
    # up to 9 products with coefficients formed in <= 3 operations, 8 additions, the normalisation (3 operations and a
    # division) and the final product: gamma(1 + 3 + 8 + 4 + 1) relative to the sum of the magnitudes
    bound = gamma(17) * mag
    return out, bound


# ---- edge-preserving filter (epf.rs, impls/generic/epf.rs) ------------------------------------------------------------

EPF_KERNEL = {0: [(0, -2), (-1, -1), (0, -1), (1, -1), (-2, 0), (-1, 0), (1, 0), (2, 0), (-1, 1), (0, 1), (1, 1), (0, 2)],
              1: [(0, -1), (0, 1), (-1, 0), (1, 0)], 2: [(0, -1), (0, 1), (-1, 0), (1, 0)]}
EPF_DIST = {0: [(0, -1), (1, 0), (0, 0), (-1, 0), (0, 1)], 1: [(0, -1), (0, 0), (0, 1), (-1, 0), (1, 0)], 2: [(0, 0)]}


class EpfParams:
    """filter.rs:81-103, 176-185 defaults (f32 constants, as the reference stores them)."""

    def __init__(self, **kw):
        self.channel_scale = [float(F32(v)) for v in (40.0, 5.0, 3.5)]
        self.pass0_sigma_scale = float(F32(0.9))
        self.pass2_sigma_scale = float(F32(6.5))
        self.border_sad_mul = float(F32(2.0 / 3.0))
        self.sigma_for_modular = 1.0
        self.__dict__.update(kw)


class EpfFaults:
    """Planted model errors for the negative controls (all off by default)."""

    def __init__(self, border_col=0, replicate=False, sigma_le=False):
        self.border_col = border_col  # 8x8 border columns x % 8 in {border_col, 7} instead of {0, 7}
        self.replicate = replicate    # clamp coordinates to the edge instead of mirroring them
        self.sigma_le = sigma_le      # copy the input where sigma <= 0.3 instead of < 0.3


def sigma_per_pixel(sigma_grid, h, w, constant=None):
    if sigma_grid is None:
        return np.full((h, w), float(F32(constant)))
    g = np.asarray(sigma_grid, dtype=np.float64)
    return g[np.arange(h)[:, None] // 8, np.arange(w)[None, :] // 8]


def epf_step(planes, sigma, step, prm, err_in=None, faults=None):
    """One step (0, 1 or 2) on three channels (float64 arrays) with per-pixel sigma. Returns (out[3], bound[3])."""
    faults = faults or EpfFaults()
    x = [np.asarray(p, dtype=np.float64) for p in planes]
    h, w = x[0].shape
    d_in = [np.zeros((h, w))] * 3 if err_in is None else [np.asarray(e, dtype=np.float64) for e in err_in]
    reach = 3
    if faults.replicate:
        def shifter(a):
            ys = np.clip(np.arange(-reach, h + reach), 0, h - 1)
            xs = np.clip(np.arange(-reach, w + reach), 0, w - 1)
            p = a[np.ix_(ys, xs)]
            return lambda dx, dy: p[reach + dy: reach + dy + h, reach + dx: reach + dx + w]
    else:
        def shifter(a):
            return _shifter(a, reach)
    sx = [shifter(c) for c in x]
    se = [shifter(e) for e in d_in]
    yy, xx = np.mgrid[0:h, 0:w]
    bc = faults.border_col
    border = ((yy % 8) == 0) | ((yy % 8) == 7) | ((xx % 8) == bc) | ((xx % 8) == 7)
    step_mul = prm.pass0_sigma_scale if step == 0 else (prm.pass2_sigma_scale if step == 2 else 1.0)
    sm = np.where(border, step_mul * prm.border_sad_mul, step_mul)
    six6 = float(F32(6.6)) * (float(F32(0.7071067811865476)) - 1.0)
    # (sigma 0 only occurs where the input is copied; any finite value serves there)
    nis = six6 / np.where(sigma > 0, sigma, 1.0) * sm
    wsum = np.ones((h, w))
    num = [c.copy() for c in x]
    ks = EPF_KERNEL[step]
    weights, dws, nbrs, nbr_err = [], [], [], []
    for kx, ky in ks:
        dist = np.zeros((h, w))
        ddist = np.zeros((h, w))
        for c in range(3):
            acc = np.zeros((h, w))
            dacc = np.zeros((h, w))
            for ix, iy in EPF_DIST[step]:
                acc += np.abs(sx[c](kx + ix, ky + iy) - sx[c](ix, iy))
                dacc += se[c](kx + ix, ky + iy) + se[c](ix, iy)
            dist += prm.channel_scale[c] * acc
            ddist += prm.channel_scale[c] * dacc
        t = dist * nis
        wk = np.maximum(0.0, 1.0 + t)
        # |d_f32 - d| <= ddist (inputs) + gamma(8) d (5 differences, 4 additions, the scale, 2 channel additions);
        # nis carries gamma(5) (subtraction, product, division, two step-multiplier products); max(0, .) is 1-Lipschitz
        dw = np.abs(nis) * (ddist + gamma(8) * dist) + gamma(7) * (1.0 + np.abs(t))
        weights.append(wk)
        dws.append(dw)
        nbrs.append([sx[c](kx, ky) for c in range(3)])
        nbr_err.append([se[c](kx, ky) for c in range(3)])
        wsum += wk
        for c in range(3):
            num[c] += wk * nbrs[-1][c]
    out = [n / wsum for n in num]
    dw_sum = sum(dws)
    w_low = np.maximum(wsum - dw_sum, 1e-300)
    n = len(ks)
    bounds = []
    for c in range(3):
        # perturbed weighted mean: (sum dw_k (|X_k - out| + D_k) + sum w_k D_k + D_centre) / (W - sum dw_k)
        pert = d_in[c].copy()
        mag = np.abs(x[c]).copy()
        for k in range(n):
            pert += dws[k] * (np.abs(nbrs[k][c] - out[c]) + nbr_err[k][c]) + weights[k] * nbr_err[k][c]
            mag += weights[k] * np.abs(nbrs[k][c])
        # f32 numerator (n products, n additions), denominator (n additions) and the division
        rnd = (gamma(2 * n + 1) * mag + gamma(n) * np.abs(out[c]) * wsum) / w_low + U * np.abs(out[c])
        bounds.append(pert / w_low + rnd)
    keep = (sigma <= float(F32(0.3))) if faults.sigma_le else (sigma < float(F32(0.3)))
    out = [np.where(keep, x[c], out[c]) for c in range(3)]
    bounds = [np.where(keep, d_in[c], bounds[c]) for c in range(3)]
    return out, bounds


def epf(planes, sigma, iters, prm=None, err_in=None, faults=None):
    """apply_epf (epf.rs:10-104): step 0 when iters == 3, step 1, step 2 when iters >= 2."""
    prm = prm or EpfParams()
    steps = ([0] if iters == 3 else []) + [1] + ([2] if iters >= 2 else [])
    out, err = planes, err_in
    for st in steps:
        out, err = epf_step(out, sigma, st, prm, err, faults)
    return out, err


# ---- XYB -> linear sRGB -> sRGB (xyb.rs, ciexyz.rs defaults, IEC 61966-2-1) --------------------------------------------

OPSIN_INV = np.array([[11.031566901960783, -9.866943921568629, -0.16462299647058826],
                      [-3.254147380392157, 4.418770392156863, -0.16462299647058826],
                      [-3.6588512862745097, 2.7129230470588235, 1.9459282392156863]], dtype=np.float32).astype(np.float64)
OPSIN_BIAS = float(F32(-0.0037930732552754493))


def xyb_to_linear(xyb, matrix=OPSIN_INV, bias=(OPSIN_BIAS,) * 3, itscale=1.0, err_in=None):
    """XybToMixedLms + Matrix (xyb.rs:35-60, convert.rs:287-308) with the f32 parameters taken as exact.
    Returns (rgb[3], bound[3])."""
    x, y, b = [np.asarray(p, dtype=np.float64) for p in xyb]
    e = [np.zeros_like(x)] * 3 if err_in is None else [np.asarray(v, dtype=np.float64) for v in err_in]
    cb = [np.cbrt(v) for v in bias]
    g = [y + x - cb[0], y - x - cb[1], b - cb[2]]
    gmag = [np.abs(y) + np.abs(x) + abs(cb[0]), np.abs(y) + np.abs(x) + abs(cb[1]), np.abs(b) + abs(cb[2])]
    # the f32 cube root of the bias is within one ulp (2u relative) of the exact one
    eg = [gamma(2) * gmag[i] + 2 * U * abs(cb[i]) for i in range(3)]
    eg = [eg[0] + e[1] + e[0], eg[1] + e[1] + e[0], eg[2] + e[2]]
    lms = [(g[i] ** 3 + bias[i]) * itscale for i in range(3)]
    # g*g, *g (fused with + bias), * itscale: 3 roundings of the magnitudes, plus the propagated |3 g^2| eg (+ eg^3 terms)
    elms = [(3 * g[i] ** 2 * eg[i] + 3 * np.abs(g[i]) * eg[i] ** 2 + eg[i] ** 3 + gamma(3) * (np.abs(g[i]) ** 3 + abs(bias[i]))) * abs(itscale)
            for i in range(3)]
    out, bound = [], []
    for r in range(3):
        o = sum(matrix[r, j] * lms[j] for j in range(3))
        mag = sum(abs(matrix[r, j]) * np.abs(lms[j]) for j in range(3))
        out.append(o)
        bound.append(gamma(3) * mag + sum(abs(matrix[r, j]) * elms[j] for j in range(3)))
    return out, bound


SRGB_THRESHOLD = 0.0031308


def srgb_exact(v, slope=12.92):
    """IEC 61966-2-1 encoding, odd extension to negative values (`slope` is a negative-control hook)."""
    v = np.asarray(v, dtype=np.float64)
    a = np.abs(v)
    return np.sign(v) * np.where(a <= SRGB_THRESHOLD, slope * a, 1.055 * np.power(a, 1 / 2.4) - 0.055)


# The exact curve's steepest slope: 12.92 on the linear segment; above the threshold 1.055 / 2.4 v^(1/2.4 - 1) < 12.92
SRGB_MAX_SLOPE = 12.92


def srgb(lin, lin_bound, approx_rel, slope=12.92):
    """The kernels' sRGB stage on values known to within lin_bound: |kernel - exact(lin)| <= r * |exact| + SRGB_MAX_SLOPE *
    lin_bound, where r = approx_rel = (r_linear, r_power) is the measured relative error of the kernels' curve on the
    segment the f32 input can lie on (both where it may lie on either)."""
    out = srgb_exact(lin, slope)
    a = np.abs(lin)
    r_lin, r_pow = approx_rel
    r = np.where(a + lin_bound <= SRGB_THRESHOLD, r_lin, np.where(a - lin_bound > SRGB_THRESHOLD, r_pow, max(r_lin, r_pow)))
    return out, r * (np.abs(out) + SRGB_MAX_SLOPE * lin_bound) + SRGB_MAX_SLOPE * lin_bound



# ---- non-separable upsampling (features/upsampling.rs:45-132, util.rs:423-454) ------------------------------------------

def _weights(name):
    """A default weight table of host/upsampling_weights.inc (the specification's constants), as the f32 values."""
    import os
    import re
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "jxl_oxide_b200", "csrc", "host",
                        "upsampling_weights.inc")
    text = open(path).read()
    body = re.search(name + r"\[\d+\] = \{(.*?)\};", text, re.S).group(1)
    return np.array([float(v.rstrip("f")) for v in re.findall(r"-?\d+\.\d+(?:e-?\d+)?f", body)], dtype=np.float32).astype(np.float64)


UP_WEIGHTS = {2: "kDefaultUp2", 4: "kDefaultUp4", 8: "kDefaultUp8"}


def _padded(x, mirror_quirk=True):
    """PaddedGrid with padding 2 after mirror_edges_padding. The reference mirrors in place, so an input one sample wide
    reads padding cells it has not written yet and leaves the outer column on each side 0 ([0, s, s, s, 0]); one sample
    high, the outermost top row stays 0. mirror_quirk=False pads with a proper mirror (a negative-control hook)."""
    h, w = x.shape
    if not mirror_quirk:
        return x[np.ix_(mirror(np.arange(-2, h + 2), h), mirror(np.arange(-2, w + 2), w))]
    pw = w + 4
    p = np.zeros((h + 4, pw))
    p[2:h + 2, 2:w + 2] = x
    for y in range(2, h + 2):
        for i in range(2):
            p[y, i] = p[y, 3 - i]
            p[y, pw - 1 - i] = p[y, pw - 4 + i]
    top = p[2:4].copy()  # split_at_mut: the rows the top padding copies, as they are before the bottom one is written
    p[0], p[1] = top[1], top[0]
    for r, src in zip((h + 2, h + 3), (h + 1, h)):
        p[r] = p[src]
    return p


def upsample(x, factor, mirror_quirk=True):
    """One channel, factor 2, 4 or 8 (one pass each): a 5x5 kernel per output phase from the symmetric weight list,
    clamped to the min / max of the 25 samples. Returns (out, bound)."""
    x = np.asarray(x, dtype=np.float64)
    h, w = x.shape
    k, n = factor, factor // 2
    wts = _weights(UP_WEIGHTS[factor])
    big = np.zeros((5 * n, 5 * n))
    idx = 0
    for y in range(5 * n):
        for xx in range(y, 5 * n):
            big[y, xx] = big[xx, y] = wts[idx]
            idx += 1
    p = _padded(x, mirror_quirk)
    win = np.stack([p[iy:iy + h, ix:ix + w] for iy in range(5) for ix in range(5)])  # (25, h, w)
    lo, hi = win.min(0), win.max(0)
    out = np.empty((h * k, w * k))
    bound = np.empty_like(out)
    for py in range(k):
        my, fv = min(py, k - py - 1), py >= n
        for px in range(k):
            mx, fh = min(px, k - px - 1), px >= n
            kern = big[my * 5:my * 5 + 5, mx * 5:mx * 5 + 5]
            kern = kern[::-1] if fv else kern
            kern = kern[:, ::-1] if fh else kern
            kv = kern.reshape(25, 1, 1)
            s = (kv * win).sum(0)
            # 25 products summed in sequence: gamma(25) of the summed magnitudes; the clamp is 1-Lipschitz
            out[py::k, px::k] = np.clip(s, lo, hi)
            bound[py::k, px::k] = gamma(25) * (np.abs(kv) * np.abs(win)).sum(0)
    return out, bound

# ---- exact integer models (rct.rs, squeeze.rs) ------------------------------------------------------------------------

def wrap32(v):
    v = np.asarray(v, dtype=np.int64)
    return ((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def rct_inverse(a, b, c, rct_type):
    """inverse_rct (rct.rs:15-140, 201-256) with wrapping i32 arithmetic; rct_type = 7 * permutation + type."""
    perm, ty = rct_type // 7, rct_type % 7
    a, b, c = [np.asarray(v, dtype=np.int64) for v in (a, b, c)]
    if ty == 6:
        tmp = wrap32(a - (c >> 1))
        e = wrap32(c + tmp)
        f = wrap32(tmp - (b >> 1))
        d = wrap32(f + b)
    else:
        d = a
        f = wrap32(c + a) if ty & 1 else c
        if ty >> 1 == 1:
            e = wrap32(b + a)
        elif ty >> 1 == 2:
            e = wrap32(b + (wrap32(a + f) >> 1))
        else:
            e = b
    order = {0: (d, e, f), 1: (f, d, e), 2: (e, f, d), 3: (d, f, e), 4: (e, d, f), 5: (f, e, d)}[perm]
    return [o.astype(np.int32) for o in order]


def _tdiv(a, b):
    return np.sign(a) * (np.abs(a) // b)


def tendency(a, b, c):
    """tendency_i32 (squeeze.rs:1104-1137): Wrapping<i32> throughout, `/` truncating."""
    a, b, c = [np.asarray(v, dtype=np.int64) for v in (a, b, c)]
    up = (a >= b) & (b >= c)
    dn = (a <= b) & (b <= c)
    x_up = wrap32(_tdiv(wrap32(wrap32(wrap32(wrap32(4 * a) - wrap32(3 * c)) - b) + 6), 12))
    t1 = wrap32(2 * wrap32(a - b))
    x_up = np.where(wrap32(x_up - (x_up & 1)) > t1, wrap32(t1 + 1), x_up)
    t2 = wrap32(2 * wrap32(b - c))
    x_up = np.where(wrap32(x_up + (x_up & 1)) > t2, t2, x_up)
    x_dn = wrap32(_tdiv(wrap32(wrap32(wrap32(wrap32(4 * a) - wrap32(3 * c)) - b) - 6), 12))
    x_dn = np.where(wrap32(x_dn + (x_dn & 1)) < t1, wrap32(t1 - 1), x_dn)
    x_dn = np.where(wrap32(x_dn - (x_dn & 1)) < t2, t2, x_dn)
    return np.where(up, x_up, np.where(dn, x_dn, 0))


def squeeze_inverse_h(avg, res):
    """inverse_h_i32_base (squeeze.rs:59-88): rows of avg (w_a) and residuals (w_r = w_a or w_a - 1) -> w_a + w_r."""
    avg = np.asarray(avg, dtype=np.int64)
    res = np.asarray(res, dtype=np.int64).reshape(avg.shape[0], -1)
    h, wa = avg.shape
    wr = res.shape[1]
    out = np.zeros((h, wa + wr), dtype=np.int64)
    cur = avg[:, 0]
    left = cur
    for x in range(wr):
        nxt = avg[:, x + 1] if x + 1 < wa else cur
        diff = wrap32(res[:, x] + tendency(left, cur, nxt))
        first = wrap32(cur + _tdiv(diff, 2))
        second = wrap32(first - diff)
        out[:, 2 * x], out[:, 2 * x + 1] = first, second
        cur, left = nxt, second
    if (wa + wr) % 2:
        out[:, -1] = avg[:, wa - 1]
    return out.astype(np.int32)


def squeeze_inverse_v(avg, res):
    """inverse_v: the same on columns."""
    return squeeze_inverse_h(np.asarray(avg).T, np.asarray(res).reshape(-1, np.asarray(avg).shape[1]).T).T.copy()
