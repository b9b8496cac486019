"""Seeded images and parameters for the JPEG encoder's tests: every case names the libjpeg-turbo rule it reaches.

`cases()` gives (name, image, params) triples, grey and BGR, made from fixed seeds, so the same bytes on every machine.
Parameters are cv2-style flat lists: IMWRITE_JPEG_QUALITY 1, OPTIMIZE 3, RST_INTERVAL 4, SAMPLING_FACTOR 7."""
import numpy as np

SEED = 20261019
Q, OPT, RST, SF = 1, 3, 4, 7
SAMPLINGS = {"411": 0x411111, "420": 0x221111, "422": 0x211111, "440": 0x121111, "444": 0x111111}
QUALITIES = (0, 1, 5, 10, 50, 75, 90, 95, 100)
RESTARTS = (0, 1, 3, 65535)


def _bgr(g, rng):
    """three different planes from one pattern, so chroma is not flat"""
    g = g.astype(np.int64)
    return np.stack([g, 255 - g, (g * 3 + rng.integers(0, 8, g.shape)) % 256], -1).astype(np.uint8)


def page(kind, h, w, c, rng):
    """flat, gradient, noise or text-like (dark strokes on paper with a little scanner noise)"""
    if kind == "flat":
        g = np.full((h, w), 201, np.uint8)
        return np.stack([g, np.full((h, w), 180, np.uint8), np.full((h, w), 90, np.uint8)], -1) if c == 3 else g
    if kind == "gradient":
        y, x = np.mgrid[0:h, 0:w]
        g = ((x * 255) // max(w - 1, 1) + (y * 97) // max(h - 1, 1)) % 256
    elif kind == "noise":
        return rng.integers(0, 256, (h, w, 3) if c == 3 else (h, w), dtype=np.uint8)
    else:
        g = np.full((h, w), 236, np.int64)
        for _ in range(max(1, h * w // 400)):
            y0, x0 = rng.integers(0, h), rng.integers(0, w)
            if rng.random() < 0.5:
                g[y0:y0 + 2, x0:x0 + rng.integers(3, 14)] = 20
            else:
                g[y0:y0 + rng.integers(3, 14), x0:x0 + 2] = 20
        g = np.clip(g + rng.integers(-6, 7, (h, w)), 0, 255)
    return _bgr(g, rng) if c == 3 else g.astype(np.uint8)


def cases(large=True):
    rng = np.random.default_rng(SEED)
    out = []
    # sizes at the edges: one pixel, one row or column 8193 long, odd sizes off every block and MCU grid
    for c in (1, 3):
        tag = "g" if c == 1 else "c"
        for h, w in ((1, 1), (1, 8193), (8193, 1), (45, 71), (17, 9), (9, 17), (31, 33)):
            img = page("noise" if h * w < 64 else "text", h, w, c, rng)
            out.append(("size%dx%d_%s" % (h, w, tag), img, []))
            out.append(("size%dx%d_%s_411_opt_rst3" % (h, w, tag), img, [SF, SAMPLINGS["411"], OPT, 1, RST, 3]))
            out.append(("size%dx%d_%s_440_rst1" % (h, w, tag), img, [SF, SAMPLINGS["440"], RST, 1]))
    # every quality on each kind of page, grey and BGR
    for kind in ("flat", "gradient", "noise", "text"):
        for c in (1, 3):
            tag = "g" if c == 1 else "c"
            img = page(kind, 45, 71, c, rng)
            for q in QUALITIES:
                out.append(("%s_%s_q%d" % (kind, tag, q), img, [Q, q]))
            # every sampling with optimise off and on (a grey image ignores the sampling)
            for sname, sv in SAMPLINGS.items():
                for opt in (0, 1):
                    out.append(("%s_%s_%s_opt%d" % (kind, tag, sname, opt), img, [SF, sv, OPT, opt]))
            for r in RESTARTS:
                out.append(("%s_%s_rst%d" % (kind, tag, r), img, [RST, r, Q, 75]))
                out.append(("%s_%s_rst%d_444_opt" % (kind, tag, r), img, [RST, r, SF, SAMPLINGS["444"], OPT, 1]))
    # q100 noise: DC and AC categories at their top (11 and 10 bits), many FF bytes to stuff
    noise = page("noise", 64, 80, 3, rng)
    for sname in ("420", "444"):
        for opt in (0, 1):
            out.append(("noise_q100_%s_opt%d" % (sname, opt), noise, [Q, 100, SF, SAMPLINGS[sname], OPT, opt]))
    out.append(("noise_q100_g_rst1", noise[..., 0].copy(), [Q, 100, RST, 1]))
    # what cv2 does with parameters out of range: clamps, and 4:2:0 for an unknown sampling value
    img = page("gradient", 23, 37, 3, rng)
    for name, p in (("q_neg", [Q, -5]), ("q_105", [Q, 105]), ("opt_2", [OPT, 2]), ("opt_neg", [OPT, -1]),
                    ("rst_70000", [RST, 70000]), ("rst_neg", [RST, -3]), ("sf_bad", [SF, 0x420])):
        out.append(("clamp_" + name, img, p))
    if large:
        big = page("text", 1170, 1654, 3, rng)
        out.append(("text_1170x1654_c", big, []))
        out.append(("text_1170x1654_c_444_opt", big, [SF, SAMPLINGS["444"], OPT, 1]))
    return out


def golden_page():
    """the golden scan decoded as the reference reads it, at the defaults and at 4:4:4 with optimised tables"""
    import os
    import cv2
    here = os.path.dirname(os.path.abspath(__file__))
    page = cv2.imdecode(np.fromfile(os.path.join(here, "golden", "AisazuNihaIrarenai-003.jpg"), np.uint8),
                        cv2.IMREAD_COLOR)
    return [("golden_page", page, []), ("golden_page_444_opt", page, [SF, SAMPLINGS["444"], OPT, 1]),
            ("golden_grey_rst8", cv2.cvtColor(page, cv2.COLOR_BGR2GRAY), [RST, 8, Q, 90])]
