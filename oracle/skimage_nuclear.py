"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

scikit-image is not installed in this container.  ``pylinac.nuclear`` (PlanarUniformity.preprocess and get_fov, nuclear.py:399-474)
calls six skimage functions; this module restates them on numpy / scipy and :func:`install` binds them into ``pylinac.nuclear`` only,
so the UNMODIFIED reference runs end to end.  The functions of oracle/skimage_shim.py keep their behaviour; none is rebound here.
Restated without the skimage source at hand (UNPINNED, like the other skimage restatements, DESIGN.md section 8.5).
"""
from __future__ import annotations

import numpy as np
from scipy import ndimage


def block_reduce(image, block_size=2, func=np.sum, cval=0, func_kwargs=None):
    """skimage.measure.block_reduce: pad the end of each axis with `cval` up to a multiple of the block, then `func` over each block
    (np.sum of uint16 blocks gives uint64)."""
    image = np.asarray(image)
    if np.isscalar(block_size):
        block_size = (block_size,) * image.ndim
    pad = [(0, (-s) % b) for s, b in zip(image.shape, block_size)]
    padded = np.pad(image, pad, mode="constant", constant_values=cval)
    hb, wb = padded.shape[0] // block_size[0], padded.shape[1] // block_size[1]
    blocks = padded.reshape(hb, block_size[0], wb, block_size[1]).transpose(0, 2, 1, 3)
    return func(blocks, axis=(2, 3), **(func_kwargs or {}))


def label(image, connectivity=None, return_num=False, background=0):
    """skimage.measure.label: raster-order labels; connectivity 1 = 4 neighbours, None / 2 = 8 neighbours"""
    structure = ndimage.generate_binary_structure(2, 1 if connectivity == 1 else 2)
    lab, num = ndimage.label(np.asarray(image) != background, structure=structure)
    return (lab, num) if return_num else lab


def regionprops(label_image, intensity_image=None, **kwargs):
    """skimage.measure.regionprops, the two properties get_fov reads: ``area`` and ``image`` (the region's bounding-box crop)"""
    from oracle.skimage_shim import regionprops as shim_regionprops

    return shim_regionprops(label_image, intensity_image)


def remove_small_objects(ar, min_size=64, connectivity=1, *, out=None):
    """skimage.morphology.remove_small_objects: zero the connected components (``connectivity`` neighbourhood) of fewer than
    `min_size` pixels; a bool input is labelled first."""
    if out is None:
        out = ar.copy()
    else:
        out[:] = ar
    if min_size == 0:
        return out
    if out.dtype == bool:
        ccs = np.zeros(ar.shape, np.int32)
        ndimage.label(ar, ndimage.generate_binary_structure(ar.ndim, connectivity), output=ccs)
    else:
        ccs = out
    sizes = np.bincount(ccs.ravel())
    out[(sizes < min_size)[ccs]] = 0
    return out


def remove_small_holes(ar, area_threshold=64, connectivity=1, *, out=None):
    """skimage.morphology.remove_small_holes: remove_small_objects on the inverse, inverted back"""
    if out is None:
        out = ar.astype(bool, copy=True)
    np.logical_not(ar, out=out)
    out = remove_small_objects(out, area_threshold, connectivity, out=out)
    np.logical_not(out, out=out)
    return out


def isotropic_erosion(image, radius, out=None, spacing=None):
    """skimage.morphology.isotropic_erosion: Euclidean distance to the nearest background pixel > radius"""
    dist = ndimage.distance_transform_edt(image, sampling=spacing)
    return np.greater(dist, radius, out=out)


def find_boundaries(label_img, connectivity=1, mode="thick", background=0):
    """skimage.segmentation.find_boundaries (modes thick / inner / outer): grey dilation != grey erosion over the
    ``connectivity`` footprint (scipy's default reflect border), restricted to the foreground for 'inner' and the background for
    'outer'."""
    label_img = np.asarray(label_img)
    if label_img.dtype == bool:
        label_img = label_img.astype(np.uint8)
    footprint = ndimage.generate_binary_structure(label_img.ndim, connectivity)
    boundaries = ndimage.grey_dilation(label_img, footprint=footprint) != ndimage.grey_erosion(label_img, footprint=footprint)
    if mode == "inner":
        boundaries &= label_img != background
    elif mode == "outer":
        boundaries &= label_img == background
    elif mode != "thick":
        raise NotImplementedError(f"find_boundaries(mode={mode!r}) is not restated")
    return boundaries


def install():
    """Bind the restated functions into the stub-imported reference's ``pylinac.nuclear`` (after import_reference())."""
    from oracle.refstub import import_reference

    import_reference()
    import pylinac.nuclear as rn

    rn.block_reduce = block_reduce
    rn.label = label
    rn.regionprops = regionprops
    rn.remove_small_objects = remove_small_objects
    rn.remove_small_holes = remove_small_holes
    rn.isotropic_erosion = isotropic_erosion
    rn.find_boundaries = find_boundaries
    return rn
