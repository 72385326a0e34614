"""Plain restatement of cdprobe_bwcurve's size ladder and per-cell summary, from the field comments of
cdprobe_bwcurve_t in include/cdprobe.h, for the tests."""
import numpy as np

MAX_SIZES = 24
MIN_SIZE = 4096


def ladder(bpp: int) -> list:
    """4096 << k for every k with 4096 << k < bpp, then bpp; more than MAX_SIZES entries (bpp > 32 GiB) is refused."""
    if bpp <= 0:
        raise ValueError("bytes_per_pair must be positive")
    sizes, s = [], MIN_SIZE
    while s < bpp:
        sizes.append(s)
        s <<= 1
    sizes.append(bpp)
    if len(sizes) > MAX_SIZES:
        raise ValueError("bytes_per_pair over 32 GiB")
    return sizes


def summary(sizes, medians):
    """(t0_ns, peak_gbps, half_bytes) of one cell from its per-size median ns (float32 values): the median of the
    smallest size; the largest size / median in bytes per ns, rounded to float32 only at the end; the smallest size
    whose rate reaches half of the unrounded peak.  A median of 0 counts as rate 0."""
    rates = [s / float(m) if m > 0 else 0.0 for s, m in zip(sizes, medians)]
    peak = max(rates)
    half = next(s for s, r in zip(sizes, rates) if r >= peak / 2)
    return float(np.float32(medians[0])), float(np.float32(peak)), half
