"""Float64 NumPy restatement of the generic constant-coefficient update `b2_linear_forward` (DESIGN §3.3e).

Conventions (those of `data_with_halo` and of the C ABI): `f` is (T,) + the allocated shape, with a halo of `halo`
on every space axis; box bounds are inclusive domain indices; a tap is (tshift, offsets, coefficient). Then

  for time in time_m .. time_M, ascending for `f.forward` (wshift = +1), descending for `f.backward` (wshift = -1):
      f[(time + wshift) % T][p] = sum_k c_k * f[(time + s_k) % T][p + o_k]      for every p in the box

Every level read is taken whole before the write (Jacobi), the halo is read as stored and only the box is written.

`mut` selects one deliberate mistake from MUTATIONS. tests/test_linear_ref.py runs the matrix inputs with each of
them to show that the inputs make that kind of kernel or recogniser bug visible far above the tolerance.
"""
import numpy as np

MUTATIONS = {
    'axes_reversed': "tap offsets applied to the axes in reverse order",
    'level_off': "the level t read one slot further from the written one, at t - wshift",
    'offset_sign': "the first nonzero offset of the first tap that has one, sign flipped",
    'box_short': "the box one point short on the high side of the last axis",
    'backward_ascending': "an update of f.backward run from time_m up instead of from time_M down",
    'drop_last_tap': "the last tap of the table dropped",
    'halo_zero': "the halo read as zero",
}


def box_slices(lo, hi, halo):
    """Index of the box in an allocated (halo-padded) slot."""
    return tuple(slice(l + halo, h + halo + 1) for l, h in zip(lo, hi))


def run(f, halo, taps, wshift, lo, hi, time_m, time_M, mut=None, dtype=np.float64):
    """K = time_M - time_m + 1 steps of the update on a copy of `f` in `dtype`; returns the copy."""
    assert mut is None or mut in MUTATIONS, mut
    F = np.array(f, dtype=dtype)
    T, nd = F.shape[0], F.ndim - 1
    taps = [(int(s), tuple(int(x) for x in o), dtype(c)) for s, o, c in taps]
    if mut == 'drop_last_tap':
        taps = taps[:-1]
    if mut == 'axes_reversed':
        taps = [(s, o[::-1], c) for s, o, c in taps]
    if mut == 'offset_sign':
        k = next(i for i, (_, o, _) in enumerate(taps) if any(o))
        s, o, c = taps[k]
        d = next(i for i, x in enumerate(o) if x)
        taps[k] = (s, o[:d] + (-o[d],) + o[d + 1:], c)
    hi = list(hi)
    if mut == 'box_short':
        hi[-1] -= 1
    box = box_slices(lo, hi, halo)
    inner = tuple(slice(halo, n - halo) for n in F.shape[1:])
    if wshift > 0 or mut == 'backward_ascending':
        times = range(time_m, time_M + 1)
    else:
        times = range(time_M, time_m - 1, -1)
    for time in times:
        levels = {}
        for s in {s for s, _, _ in taps}:
            src = F[(time + s - (wshift if mut == 'level_off' and s == 0 else 0)) % T]
            if mut == 'halo_zero':
                z = np.zeros_like(src)
                z[inner] = src[inner]
                src = z
            levels[s] = src.copy()
        acc = np.zeros(tuple(b.stop - b.start for b in box), dtype=dtype)
        for s, o, c in taps:
            acc += c * levels[s][tuple(slice(b.start + x, b.stop + x) for b, x in zip(box, o))]
        F[(time + wshift) % T][box] = acc
    return F
