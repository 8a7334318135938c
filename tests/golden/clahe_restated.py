"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

skimage.exposure.equalize_adapthist, which the reference's light / rad phantoms apply to BBs near the field edge
(planar_imaging.py:1436-1449), restated for 2-D grey images.  ``install()`` puts it, together with the restated label / clear_border /
regionprops of oracle/skimage_shim.py, into the stub-imported reference so that the UNMODIFIED light / rad code runs end to end
(tests/golden/make_lightrad_golden.py).  Parity with scikit-image itself is UNPINNED.
"""
from __future__ import annotations

import types

import numpy as np

# skimage.exposure.equalize_adapthist (Zuiderveld's contrast-limited adaptive histogram equalisation), restated step by step from
# scikit-image's published algorithm for 2-D grey images.  UNPINNED: scikit-image is not installed, so the restatement has never
# been compared with the library itself.  Steps, in the library's order:
#   img_as_uint (floats in [-1, 1]: rint(x * 65535)), rescale_intensity to (0, 2**14 - 1) and np.round -> uint16;
#   reflect padding to whole kernels (k // 2 before, up to a multiple of k plus ceil(k / 2) after);
#   lut = arange(2**14) // (1 + 2**14 // nbins); one nbins histogram per contextual region of the padded image;
#   clip at int(max(clip_limit * k * k, 1)) and redistribute the excess (clip_histogram);
#   map = int(min(cumsum(hist) * ((2**14 - 1) / (k * k)), 2**14 - 1));
#   bilinear interpolation of the four neighbouring maps (edge-padded) with the weights r / k, 1 - r / k, accumulated in float32 in the
#   order (0, 0), (0, 1), (1, 0), (1, 1) and cast back to uint16; then astype(float64) and rescale_intensity to [0, 1].
NR_OF_GRAY = 2 ** 14


def _img_as_uint(image):
    image = np.asarray(image)
    if image.dtype == np.uint16:
        return image
    if image.dtype.kind != "f":
        raise TypeError(f"equalize_adapthist restatement: unsupported dtype {image.dtype}")
    if image.min() < -1.0 or image.max() > 1.0:
        raise ValueError("Images of type float must be between -1 and 1.")
    out = np.multiply(image, 65535, dtype=np.float64)
    np.rint(out, out=out)
    np.clip(out, 0, 65535, out=out)
    return out.astype(np.uint16)


def _rescale_intensity(image, out_range):
    """rescale_intensity(image, in_range='image', out_range): (clip(x) - imin) / (imax - imin) * (omax - omin) + omin"""
    imin, imax = float(image.min()), float(image.max())
    omin, omax = out_range
    image = np.clip(image, imin, imax)
    if imin != imax:
        image = (image - imin) / (imax - imin)
        return np.asarray(image * (omax - omin) + omin, dtype=np.float64)
    return np.clip(image, omin, omax).astype(np.float64)


def clip_histogram(hist, clip_limit):
    """Clip one histogram at clip_limit and hand the excess back to the bins below it (skimage.exposure._adapthist.clip_histogram)."""
    excess_mask = hist > clip_limit
    excess = hist[excess_mask]
    n_excess = excess.sum() - excess.size * clip_limit
    hist[excess_mask] = clip_limit
    bin_incr = n_excess // hist.size
    upper = clip_limit - bin_incr
    low_mask = hist < upper
    n_excess -= hist[low_mask].size * bin_incr
    hist[low_mask] += bin_incr
    mid_mask = np.logical_and(hist >= upper, hist < clip_limit)
    mid = hist[mid_mask]
    n_excess += mid.sum() - mid.size * clip_limit
    hist[mid_mask] = clip_limit
    while n_excess > 0:
        prev_n_excess = n_excess
        for index in range(hist.size):
            under_mask = hist < clip_limit
            step_size = max(1, np.count_nonzero(under_mask) // n_excess)
            under_mask = under_mask[index::step_size]
            hist[index::step_size][under_mask] += 1
            n_excess -= np.count_nonzero(under_mask)
            if n_excess <= 0:
                break
        if prev_n_excess == n_excess:
            break
    return hist


def map_histogram(hist, min_val, max_val, n_pixels):
    out = np.cumsum(hist, axis=-1).astype(float)
    out *= (max_val - min_val) / n_pixels
    out += min_val
    np.clip(out, a_min=None, a_max=max_val, out=out)
    return out.astype(int)


def clahe_u14(image14, k: int, clip_limit: float = 0.01, nbins: int = 256):
    """The contextual-region part of CLAHE on a 2-D uint16 image of 14-bit values -> uint16 (before the final rescale)."""
    h, w = image14.shape
    ps = k // 2
    pe = [(k - s % k) % k + int(np.ceil(k / 2.0)) for s in (h, w)]
    img = np.pad(image14, [[ps, pe[0]], [ps, pe[1]]], mode="reflect")
    bin_size = 1 + NR_OF_GRAY // nbins
    lut = np.arange(NR_OF_GRAY, dtype=np.uint16) // bin_size
    img = lut[img]
    nh = [int(s / k) - 1 for s in img.shape]
    blocks = img[ps:ps + nh[0] * k, ps:ps + nh[1] * k].reshape(nh[0], k, nh[1], k).transpose(0, 2, 1, 3).reshape(nh[0] * nh[1], -1)
    kernel_elements = k * k
    clim = int(np.clip(clip_limit * kernel_elements, 1, None)) if clip_limit > 0.0 else kernel_elements
    hist = np.stack([np.bincount(b, minlength=nbins) for b in blocks])
    hist = np.stack([clip_histogram(hh, clim) for hh in hist])
    hist = map_histogram(hist, 0, NR_OF_GRAY - 1, kernel_elements).reshape(nh[0], nh[1], -1)
    map_array = np.pad(hist, [[1, 1], [1, 1], [0, 0]], mode="edge")
    npr = [int(s / k) for s in img.shape]
    pb = img.reshape(npr[0], k, npr[1], k).transpose(0, 2, 1, 3).reshape(npr[0] * npr[1], k * k)
    frac = np.arange(k) / k
    col = np.tile(frac, k)                 # coefficient of the column offset inside a block (flattened row-major)
    row = np.repeat(frac, k)
    coeffs = [col, row]
    inv_coeffs = [1 - c for c in coeffs]
    result = np.zeros(pb.shape, dtype=np.float32)
    for edge in np.ndindex(2, 2):
        edge_maps = map_array[edge[0]:edge[0] + npr[0], edge[1]:edge[1] + npr[1]].reshape(npr[0] * npr[1], -1)
        edge_mapped = np.take_along_axis(edge_maps, pb.astype(np.int64), axis=-1)
        edge_coeffs = np.prod([[inv_coeffs, coeffs][e][d] for d, e in enumerate(edge[::-1])], 0)
        result += (edge_mapped * edge_coeffs).astype(result.dtype)
    result = result.astype(np.uint16)
    result = result.reshape(npr[0], npr[1], k, k).transpose(0, 2, 1, 3).reshape(img.shape)
    return result[ps:img.shape[0] - pe[0], ps:img.shape[1] - pe[1]]


def equalize_adapthist(image, kernel_size=None, clip_limit=0.01, nbins=256):
    """skimage.exposure.equalize_adapthist for a 2-D grey image (restated, unpinned; see the block comment above)."""
    image = _img_as_uint(image)
    image = np.round(_rescale_intensity(image, (0, NR_OF_GRAY - 1))).astype(np.uint16)
    if kernel_size is None:
        kernel_size = max(image.shape[0] // 8, 1)
    if not np.isscalar(kernel_size):
        if len(set(int(k) for k in kernel_size)) != 1:
            raise NotImplementedError("equalize_adapthist restatement: square kernels only")
        kernel_size = kernel_size[0]
    out = clahe_u14(image, int(kernel_size), clip_limit, nbins)
    return _rescale_intensity(out.astype(np.float64), (0.0, 1.0))


def install():
    """oracle.skimage_shim.install(), then ``exposure`` of the reference's planar_imaging module -> this restatement"""
    from oracle import skimage_shim

    skimage_shim.install()
    import pylinac.planar_imaging as rplanar

    rplanar.exposure = types.SimpleNamespace(equalize_adapthist=equalize_adapthist)
