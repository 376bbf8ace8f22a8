"""Model of the slab walk of paint_kernel<_, true> (forma_b200/csrc/kernels_painter.cu
of an earlier round): walking a tile in eight two-column slabs with one
running cover per row — flat coverage left and right of the entry's segment columns — gives
the coverage of every pixel that the reference's column sweep gives
(cpu/painter/mod.rs:388-404: area(x, y) = 32 * sum of covers left of x + areas[x][y], covers
wrapping at i8, areas at i16). Pure NumPy; it pins the arithmetic of the walk, not the kernel."""
import numpy as np


def i8(v):
    return ((v + 128) % 256) - 128


def i16(v):
    return ((v + 32768) % 65536) - 32768


def coverage(doubled, even_odd):  # cpu/painter/mod.rs:77-94
    if not even_odd:
        return np.clip(np.abs(doubled / 512.0), 0.0, 1.0)
    return (512 - np.abs((doubled & 1023) - 512)) / 512.0


def column_sweep(area, cover, carry, even_odd):
    out = np.zeros((16, 16))
    for y in range(16):
        run = i8(int(carry[y]))
        for x in range(16):
            out[x, y] = coverage(32 * run + i16(int(area[x, y])), even_odd)
            run = i8(run + i8(int(cover[x, y])))
    return out


def slab_walk(area, cover, carry, even_odd, x_lo, x_hi):
    out = np.zeros((16, 16))
    has_cells = x_lo <= x_hi
    first, last = x_lo >> 1, x_hi >> 1
    run = [i8(int(c)) for c in carry]
    flat = [coverage(32 * r, even_odd) for r in run]
    for j in range(8):
        if has_cells and first <= j <= last:
            for par in range(2):
                for row in range(16):
                    here = i8(run[row] + (i8(int(cover[2 * j, row])) if par else 0))
                    out[2 * j + par, row] = coverage(32 * here + i16(int(area[2 * j + par, row])), even_odd)
            run = [i8(run[r] + i8(int(cover[2 * j, r])) + i8(int(cover[2 * j + 1, r]))) for r in range(16)]
            if j == last:
                flat = [coverage(32 * r, even_odd) for r in run]
        else:
            out[2 * j, :] = flat
            out[2 * j + 1, :] = flat
    return out


def test_slab_walk_equals_column_sweep():
    rng = np.random.default_rng(1)
    for trial in range(600):
        n = int(rng.integers(0, 60))
        lo, hi = sorted(int(v) for v in rng.integers(0, 16, 2))
        lx, ly = rng.integers(lo, hi + 1, n), rng.integers(0, 16, n)
        cv, dam = rng.integers(-16, 17, n), rng.integers(0, 33, n)
        scale = 40 if trial % 5 == 0 else 1          # large values exercise the i8 / i16 wrap-around
        carry = rng.integers(-3, 4, 16) * scale if trial % 3 else np.zeros(16, int)
        area, cover = np.zeros((16, 16), int), np.zeros((16, 16), int)
        for x, y, c, d in zip(lx, ly, cv, dam):
            area[x, y] += int(d) * int(c) * scale
            cover[x, y] += int(c) * scale
        x_lo, x_hi = (int(lx.min()), int(lx.max())) if n else (16, 0)
        for even_odd in (False, True):
            assert np.array_equal(column_sweep(area, cover, carry, even_odd),
                                  slab_walk(area, cover, carry, even_odd, x_lo, x_hi)), trial
