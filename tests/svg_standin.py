"""A stand-in for resvg in the SVG image tests: a deterministic rasteriser of two shapes of the reference's
integration-tests/assets/image.svg (intrinsic size 666 x 524), the sky rectangle (M1.82758 1.79309 to 664.172 522.207,
#C3E1ED) and the sun disc (centre 179.241, 126.799, radius 77.6955, #ED8A19), drawn at any resolution with the scale
(w / 666, h / 524) of render_to_texture.  Coverage is 4 x 4 supersampled, so the edges are translucent; the result is
premultiplied RGBA8, as tiny-skia's Pixmap holds it.  Test infrastructure.
"""
import numpy as np

SIZE = (666, 524)
SKY = (1.82758, 1.79309, 664.172, 522.207), (0xC3, 0xE1, 0xED)
SUN = (179.241, 126.799, 77.6955), (0xED, 0x8A, 0x19)


def rasterize(w, h, size=SIZE):
    """the two shapes drawn at w x h: an (h, w, 4) uint8 premultiplied array"""
    sx, sy = w / size[0], h / size[1]
    cov_sky, cov_sun = np.zeros((h, w)), np.zeros((h, w))
    for i in range(4):
        for j in range(4):
            # the subsample's position in SVG units
            px = (np.arange(w)[None, :] + (i + 0.5) / 4) / sx
            py = (np.arange(h)[:, None] + (j + 0.5) / 4) / sy
            (x0, y0, x1, y1), _ = SKY
            cov_sky += ((px >= x0) & (px < x1) & (py >= y0) & (py < y1)) / 16.0
            (cx, cy, r), _ = SUN
            cov_sun += ((px - cx) ** 2 + (py - cy) ** 2 < r * r) / 16.0
    rgba = np.zeros((h, w, 4))
    for cov, (_, colour) in ((cov_sky, SKY), (cov_sun, SUN)):   # source-over, in paint order
        src = np.concatenate([np.array(colour) / 255.0, [1.0]])
        rgba = src[None, None, :] * cov[..., None] + rgba * (1.0 - cov[..., None])
    return np.rint(rgba * 255.0).astype(np.uint8)
