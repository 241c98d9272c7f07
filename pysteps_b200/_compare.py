"""The dtype NumPy compares a field with a threshold in, shared by every method that thresholds a field
on the device.

NumPy 2 types a comparison by NEP 50: a Python float or int is weak and takes the field's dtype (a
float32 field is compared with float32(threshold)), an ``np.float64`` or a 0-d float64 array is strong
(compared in float64), and so are the elements of an ndarray of thresholds.  The kernels compare in
double, so the host rounds the threshold to the comparison dtype first; a float32 value widens
exactly and the result is the one NumPy gets.
"""
import numpy as np


def comparison_threshold(field_dtype, threshold, who):
    """(t, ct): ``float(threshold)`` rounded to ct = ``np.result_type(field, threshold)``, for a field
    of `field_dtype` (float32 or float64).  A threshold whose comparison dtype is neither float32 nor
    float64 raises NotImplementedError naming `who`."""
    ct = np.result_type(np.zeros(1, dtype=field_dtype), threshold)
    if ct not in (np.float32, np.float64):
        raise NotImplementedError(f"pysteps_b200 {who}: a threshold of type {type(threshold)} is not supported")
    return float(np.asarray(threshold).astype(ct)), ct
