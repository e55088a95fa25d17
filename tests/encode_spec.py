"""An independent model of what an encode writes, for the configurations the compiled reference has no planar path for.

The C restatement (oracle/avif_oracle.c) and the kernels were written from the same definitions, so a mistake they share
passes every parity test.  This model is built from other material only, and never loads the restatement:

  stage A, host pixel -> R'G'B'(A) codes:
    * where the reference has the path (integer hosts; float hosts with PQ, SMPTE 428 or no curve), the compiled
      reference's own encoder in its interleaved layout.  16-bit host samples are clamped to 32768 first: the reference
      reads past its 32769-entry table above that, and the project's definition ("the LUT formula continues and
      clamps") gives the code of 32768 for every larger sample.
    * the steps include/avifgpu.h adds (the colour-profile row matrix, the HLG save path, Gray16 -> SMPTE 428, and
      non-finite float samples the reference's cast leaves undefined) composed from the compiled reference's scalar
      functions in numpy float32, in the order the header states.  numpy does not contract a*b+c, so this is exact.
  stage B, codes -> planes, in float64: kr / kb from the reference's coefficient table, the H.273 full-range
    equations, the BOX (mean of the samples a site has) or TOP_LEFT down-filter, round half up, plus 2^(depth-1) on
    chroma; the identity matrix (GBR) passes the codes through.

Comparison: planes that are stage-A codes (the reference layout, alpha, GBR) must be equal bit for bit.  Y / Cb / Cr
must be equal wherever the float64 value is at least MARGIN codes from a rounding boundary, and within one code
elsewhere (the kernels round in float32: < 1e-3 code at 12 bits).  Every code must lie in [0, 2^depth - 1] -- a
saturated red or blue chroma site lands exactly on the boundary 2^depth - 0.5, so only the range check sees a missing
clip there.

extreme_rows() fills every chroma site with one RGB cube corner at the host's top value (or beyond it), the inputs
where the kernels' shortcuts (no upper luma clamp, one packed min on chroma) decide the result."""
import numpy as np

import oracle
from avifgpu import abi

F32 = np.float32
MARGIN = 0.01


def load():
    """The compiled reference (oracle/_ref/libavifref.so), or None where it has not been built."""
    return oracle.load_reference()


def _top(desc):
    return (1 << desc.image_bit_depth) - 1


def _quantise(v, top):
    """The float quantiser: trunc(clamp(v * max, 0, max)), NaN -> 0."""
    scaled = np.asarray(v, F32) * F32(top)
    scaled = np.where(scaled < 0, F32(0), np.where(scaled > top, F32(top), scaled))
    return np.trunc(np.where(np.isnan(scaled), F32(0), scaled)).astype(np.int64)


def _reference_codes(ref, desc, rows):
    """(H, W, C) codes from the reference's own encoder in its layout: R, G, B(, A) or Y(, A)."""
    h, w, ch = desc.height, desc.width, desc.host_channels
    if desc.host_depth == 16:
        rows = np.minimum(rows, 32768).astype(np.uint16)
    d = desc.copy(layout=abi.LAYOUT_REFERENCE, row_matrix_enabled=0, hlg_extension=0, gray16_curve=abi.GRAY16_LUT)
    planes = ref.encode(d, rows)
    if ch <= 2:
        return np.stack([planes[0]] + ([planes[3]] if ch == 2 else []), -1).astype(np.int64)
    return planes[0].reshape(h, w, ch).astype(np.int64)


def _composed_float_codes(ref, desc, rows):
    """Float RGB(A) hosts through the header's order: row matrix, alpha clamp and premultiply, HLG inverse OOTF, curve,
    quantiser -- each step a scalar of the compiled reference or one float32 operation."""
    h, w, ch = desc.height, desc.width, desc.host_channels
    top = _top(desc)
    px = rows.reshape(h, w, ch).astype(F32)
    colour = px[..., :3].copy()
    if desc.row_matrix_enabled:
        m = [F32(v) for v in desc.row_matrix]
        r, g, b = colour[..., 0].copy(), colour[..., 1].copy(), colour[..., 2].copy()
        for k in range(3):
            colour[..., k] = ((m[3 * k] * r) + (m[3 * k + 1] * g)) + (m[3 * k + 2] * b)
    alpha = None
    if ch == 4:
        a = px[..., 3]
        alpha = np.where(a < 0, F32(0), np.where(a > 1, F32(1), a)).astype(F32)
        if desc.alpha_state == abi.ALPHA_PREMULTIPLIED:
            clamped = np.where(colour < 0, F32(0), np.where(colour > 1, F32(1), colour)).astype(F32)
            product = (clamped * alpha[..., None]).astype(F32) / F32(1)
            colour = np.where((alpha < 1)[..., None], np.where((alpha == 0)[..., None], F32(0), product), colour).astype(F32)
    flat = colour.reshape(-1, 3)
    if desc.transfer == abi.TRANSFER_HLG:
        if desc.hlg_extension == abi.HLG_INVERSE_OOTF_THEN_OETF:
            flat = ref.hlg_inverse_ootf(flat, desc.nclx.color_primaries, desc.hlg_display_gamma, float(desc.hlg_peak_nits))
        curved = ref.transfer(abi.FN_LINEAR_TO_HLG, flat)
    elif desc.transfer == abi.TRANSFER_PQ:
        curved = ref.transfer(abi.FN_LINEAR_TO_PQ, flat, float(desc.pq_peak_nits))
    elif desc.transfer == abi.TRANSFER_SMPTE428:
        curved = ref.transfer(abi.FN_LINEAR_TO_SMPTE428, flat)
    else:
        curved = flat
    codes = _quantise(curved.reshape(h, w, 3), top)
    if alpha is not None:
        codes = np.concatenate([codes, _quantise(alpha, top)[..., None]], -1)
    return codes


def _gray16_smpte428_codes(ref, desc, rows):
    """Gray16 -> SMPTE 428: the reference's LinearToSMPTE428 of v / 32768 and the float quantiser; alpha by the depth
    table formula, taken from the reference's own Gray16 encoder."""
    h, w, ch = desc.height, desc.width, desc.host_channels
    px = rows.reshape(h, w, ch)
    v = (px[..., 0].astype(F32) / F32(32768)).astype(F32)
    y = _quantise(ref.transfer(abi.FN_LINEAR_TO_SMPTE428, v.reshape(-1)).reshape(h, w), _top(desc))
    if ch == 1:
        return y[..., None]
    return np.stack([y, _reference_codes(ref, desc, rows)[..., 1]], -1)


def stage_a(ref, desc, rows):
    """(H, W, C) integer codes of every host pixel: R, G, B(, A) for RGB(A) hosts, Y(, A) for Gray(A) hosts."""
    if desc.host_depth == 16 and desc.host_channels <= 2 and desc.gray16_curve == abi.GRAY16_SMPTE428:
        return _gray16_smpte428_codes(ref, desc, rows)
    if desc.host_depth == 32 and (desc.transfer == abi.TRANSFER_HLG or desc.row_matrix_enabled or not np.isfinite(rows).all()):
        assert desc.host_channels in (3, 4), "the model composes RGB(A) float hosts only"
        return _composed_float_codes(ref, desc, rows)
    return _reference_codes(ref, desc, rows)


def _down(c, xs, ys, top_left):
    h, w = c.shape
    if top_left:
        return c[::1 << ys, ::1 << xs]
    ch, cw = (h + ys) >> ys, (w + xs) >> xs
    total, count = np.zeros((ch, cw)), np.zeros((ch, cw))
    for dy in range(1 << ys):
        for dx in range(1 << xs):
            part = c[dy::1 << ys, dx::1 << xs]
            total[:part.shape[0], :part.shape[1]] += part
            count[:part.shape[0], :part.shape[1]] += 1
    return total / count


def stage_b(ref, desc, codes):
    """Planar YCbCr from stage-A codes: [Y, Cb, Cr] as float64 values before rounding (None for pass-through planes)."""
    nclx = desc.nclx if desc.nclx.present else None
    r, g, b = (codes[..., i].astype(np.float64) for i in range(3))
    if nclx is not None and nclx.matrix_coefficients == abi.MATRIX_GBR:
        return [None, None, None], [g, b, r], 0
    kr, kg, kb = ref.yuv_coefficients(nclx).astype(np.float64)
    y = kr * r + kg * g + kb * b
    cb = (b - y) / (2 * (1 - kb))
    cr = (r - y) / (2 * (1 - kr))
    offset = 1 << (desc.image_bit_depth - 1)
    return [y, cb, cr], None, offset


class Expected:
    """The model's planes for one description and input: `codes[k]` (int64, or None where the plane is absent) and
    `exact[k]`, the float64 value before rounding for Y / Cb / Cr (None where the plane must match bit for bit)."""

    def __init__(self, ref, desc, rows):
        self.desc = desc
        self.top = _top(desc)
        a = stage_a(ref, desc, rows)
        h, w = desc.height, desc.width
        self.codes, self.exact = [None] * 4, [None] * 4
        has_alpha = desc.alpha_state != abi.ALPHA_NONE
        if desc.layout == abi.LAYOUT_REFERENCE:
            if desc.host_channels <= 2:
                self.codes[0] = a[..., 0]
                if has_alpha:
                    self.codes[3] = a[..., 1]
            else:
                self.codes[0] = a.reshape(h, w * desc.host_channels)
            return
        xs, ys = abi.chroma_shifts(desc.chroma)
        top_left = desc.down_filter == abi.DOWN_FILTER_TOP_LEFT
        values, passthrough, offset = stage_b(ref, desc, a)
        if passthrough is not None:
            self.codes[0] = a[..., 1]
            for k in (1, 2):
                sub = _down(passthrough[k], xs, ys, top_left)
                if xs or ys:  # a sub-sampled identity matrix still averages
                    self.exact[k] = sub
                    self.codes[k] = np.clip(np.floor(sub + 0.5), 0, self.top).astype(np.int64)
                else:
                    self.codes[k] = sub.astype(np.int64)
        else:
            self.exact[0] = values[0]
            self.exact[1] = _down(values[1], xs, ys, top_left) + offset
            self.exact[2] = _down(values[2], xs, ys, top_left) + offset
            for k in range(3):
                self.codes[k] = np.clip(np.floor(self.exact[k] + 0.5), 0, self.top).astype(np.int64)
        if has_alpha:
            self.codes[3] = a[..., 3]

    def mismatches(self, got):
        """Human-readable reasons `got` (a list of 4 arrays / None) breaks the rule; empty when it keeps it."""
        out = []
        for k, want in enumerate(self.codes):
            plane = got[k] if k < len(got) else None
            if (want is None) != (plane is None):
                out.append(f"plane {k}: present {plane is not None}, expected {want is not None}")
                continue
            if want is None:
                continue
            g = np.asarray(plane).astype(np.int64)
            if g.shape != want.shape:
                out.append(f"plane {k}: shape {g.shape}, expected {want.shape}")
                continue
            outside = (g < 0) | (g > self.top)
            if outside.any():
                at = tuple(np.argwhere(outside)[0])
                out.append(f"plane {k}: {int(outside.sum())} codes outside [0, {self.top}], first {g[at]} at {at}")
                continue
            diff = np.abs(g - want)
            if self.exact[k] is None:
                if diff.any():
                    at = tuple(np.argwhere(diff != 0)[0])
                    out.append(f"plane {k}: {int((diff != 0).sum())} codes differ, first at {at}: {g[at]} expected {want[at]}")
                continue
            v = self.exact[k] + 0.5
            frac = v - np.floor(v)
            near = np.minimum(frac, 1 - frac) < MARGIN
            bad = (diff > 1) | ((diff != 0) & ~near)
            if bad.any():
                at = tuple(np.argwhere(bad)[0])
                out.append(f"plane {k}: {int(bad.sum())} codes break the rule, first at {at}: {g[at]} expected {want[at]} "
                           f"(value {self.exact[k][at]:.6f})")
        return out


def assert_matches(ref, desc, rows, got, what=""):
    problems = Expected(ref, desc, rows).mismatches(got)
    assert not problems, f"{what}: " + "; ".join(problems)


# ---- inputs --------------------------------------------------------------------------------------------------------------

CORNERS = [(r, g, b) for r in (0, 1) for g in (0, 1) for b in (0, 1)]


def extreme_rows(desc, w, h, seed):
    """(h, w * channels) host rows whose every chroma site (2x2 in 4:2:0, 2x1 in 4:2:2, one pixel in 4:4:4) is one RGB
    cube corner at the host's top value, or beyond it (16-bit: 65535; float: >= 125.0, where PQ at 80 nits reaches the
    top code).  The corner steps by one site along a row and by three down a column, so every corner appears in every
    stretch of 8 sites in both directions: in the tuned interior, the right strip and the odd last row alike.  Alpha is
    0, the top value or half of it."""
    rng = np.random.default_rng(int.from_bytes(seed.encode(), "little") % 2 ** 32 if isinstance(seed, str) else seed)
    xs, ys = abi.chroma_shifts(desc.chroma) if desc.layout == abi.LAYOUT_PLANAR_YCBCR else (0, 0)
    ch = desc.host_channels
    dtype = abi.host_dtype(desc.host_depth)
    top, beyond, half = {8: (255, (255,), 127), 16: (32768, (65535, 40000), 16384), 32: (1.0, (125.0, 1000.0), 0.5)}[desc.host_depth]
    sites_x, sites_y = (w + xs) >> xs, (h + ys) >> ys
    start = int(rng.integers(8))
    corner = (np.arange(sites_x)[None, :] + 3 * np.arange(sites_y)[:, None] + start) % 8
    scale = np.where(rng.random((sites_y, sites_x)) < 0.7, top, rng.choice(beyond, (sites_y, sites_x)))
    site_rgb = np.asarray(CORNERS, np.float64)[corner] * scale[..., None]
    px = np.repeat(np.repeat(site_rgb, 1 << ys, 0), 1 << xs, 1)[:h, :w]
    out = np.zeros((h, w, ch), np.float64)
    colours = 1 if ch <= 2 else 3
    out[..., :colours] = px[..., :colours] if colours == 3 else px[..., 2:3]
    if ch in (2, 4):
        site_alpha = rng.choice(np.array([0, top, half], np.float64), (sites_y, sites_x))
        out[..., -1] = np.repeat(np.repeat(site_alpha, 1 << ys, 0), 1 << xs, 1)[:h, :w]
    return np.ascontiguousarray(out.astype(dtype).reshape(h, w * ch))
