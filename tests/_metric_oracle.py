"""medpy.metric.binary's dc / jc / hd95 / asd with voxelspacing (connectivity 1) restated on scipy: the reference the GPU surface
metrics (wsl4mis_b200.metric) are tested against.  medpy itself is not installed; its __surface_distances is
binary_erosion + distance_transform_edt(sampling=voxelspacing) + np.percentile / np.mean, as below."""
import numpy as np
from scipy.ndimage import binary_erosion, distance_transform_edt, generate_binary_structure


def _normalize(voxelspacing, ndim):
    if voxelspacing is None:
        return None
    sp = np.asarray(voxelspacing, dtype=np.float64)
    if sp.ndim == 0:
        return np.full(ndim, float(sp))
    if sp.shape != (ndim,):
        raise RuntimeError("sequence argument must have length equal to input rank")
    return sp


def surface(mask):
    """mask ^ binary_erosion(mask, generate_binary_structure(ndim, 1)), border_value 0."""
    mask = np.atleast_1d(np.asarray(mask).astype(bool))
    return mask ^ binary_erosion(mask, structure=generate_binary_structure(mask.ndim, 1), iterations=1)


def surface_distances(result, reference, voxelspacing=None):
    result = np.atleast_1d(np.asarray(result).astype(bool))
    reference = np.atleast_1d(np.asarray(reference).astype(bool))
    sp = _normalize(voxelspacing, result.ndim)
    if 0 == np.count_nonzero(result):
        raise RuntimeError('The first supplied array does not contain any binary object.')
    if 0 == np.count_nonzero(reference):
        raise RuntimeError('The second supplied array does not contain any binary object.')
    dt = distance_transform_edt(~surface(reference), sampling=sp)
    return dt[surface(result)]


def dc(result, reference):
    result, reference = np.asarray(result).astype(bool), np.asarray(reference).astype(bool)
    inter = int(np.count_nonzero(result & reference))   # Python ints: medpy's ZeroDivisionError rule, not numpy's nan
    try:
        return 2. * inter / float(int(np.count_nonzero(result)) + int(np.count_nonzero(reference)))
    except ZeroDivisionError:
        return 0.0


def jc(result, reference):
    result, reference = np.asarray(result).astype(bool), np.asarray(reference).astype(bool)
    return float(np.count_nonzero(result & reference)) / float(np.count_nonzero(result | reference))


def hd95(result, reference, voxelspacing=None):
    d1 = surface_distances(result, reference, voxelspacing)
    d2 = surface_distances(reference, result, voxelspacing)
    return np.percentile(np.hstack((d1, d2)), 95)


def asd(result, reference, voxelspacing=None):
    return surface_distances(result, reference, voxelspacing).mean()
