"""Writes forma_b200/csrc/srgb_decode.h: the sRGB8 decode table D of frames rendered over a
background (forma_renderer_render_over_device).

D[b] is the f32 nearest the standard sRGB EOTF of b / 255 when the project's encoder
(linear_to_srgb + to_byte, here through the oracle's fo_linear_to_srgb8) turns it back into b;
otherwise it is the f32 nearest that value among those the encoder turns into b. Every byte then
round-trips, so a pixel that nothing covers comes back unchanged. Needs the oracle's linear library
(oracle/linear.mk).

    python tools/make_srgb_decode.py
"""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "forma_b200", "csrc", "srgb_decode.h")


def encoder():
    """bytes = encode(values): compute_srgb's encode of colour values (f32 array) by the oracle."""
    lib = C.CDLL(os.path.join(ROOT, "oracle", "libforma_oracle_linear.so"))
    fn = lib.fo_linear_to_srgb8
    fn.restype = None
    fn.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32), C.c_void_p, C.c_uint64]
    ch = (C.c_uint32 * 4)(0, 0, 0, 0)  # every value a red channel: linear_to_srgb, then to_byte

    def encode(values):
        v = np.ascontiguousarray(np.asarray(values, np.float32).reshape(-1))
        pad = (-len(v)) % 4
        f = np.concatenate([v, np.zeros(pad, np.float32)])
        out = np.zeros(len(f), np.uint8)
        fn(f.ctypes.data, len(f) // 4, f.nbytes, 1, ch, out.ctypes.data, out.nbytes)
        return out[:len(v)]
    return encode


def eotf(b: int) -> float:
    c = b / 255.0
    return c / 12.92 if c <= 0.04045 else ((c + 0.055) / 1.055) ** 2.4


def table(encode, search_ulps: int = 1 << 20) -> np.ndarray:
    d = np.zeros(256, np.float32)
    for b in range(256):
        e = eotf(b)
        f = np.float32(e)
        if encode([f])[0] == b:
            d[b] = f
            continue
        bits = np.int64(f.view(np.int32))
        cand = (bits + np.arange(-search_ulps, search_ulps + 1, dtype=np.int64)).astype(np.int32).view(np.float32)
        ok = cand[encode(cand) == b]
        if not len(ok):
            raise SystemExit(f"no f32 within {search_ulps} ulps of the EOTF encodes to byte {b}")
        d[b] = ok[np.argmin(np.abs(ok.astype(np.float64) - e))]
    return d


def hexf(v) -> str:
    """A C hex float literal of the f32 v, without trailing zero digits."""
    mant, exp = float(v).hex().split("p")
    mant = mant.rstrip("0")
    return f"{mant}0p{exp}f" if mant.endswith(".") else f"{mant}p{exp}f"


def main() -> None:
    d = table(encoder())
    rows = []
    for i in range(0, 256, 4):
        rows.append("    " + ", ".join(hexf(v) for v in d[i:i + 4]) + ",")
    fixed = [b for b in range(256) if np.float32(eotf(b)) != d[b]]
    text = f"""// The sRGB8 decode table of frames rendered over a background (forma_renderer_render_over_device):
// D[b] is the f32 nearest the standard sRGB EOTF of b / 255 when compute_srgb's encode
// (linear_to_srgb, to_byte) turns it back into b, and otherwise the f32 nearest that value among
// those it turns into b. Every byte round-trips. Bytes of the second kind: {', '.join(map(str, fixed))}. The EOTF of
// 11 / 255 (0.0033465...) encodes to 12, because the encoder's polynomial branch reaches byte 11
// just above its linear branch's end at 0.0031308.
// Written by tools/make_srgb_decode.py with the oracle's encoder; tests/test_over_oracle.py pins it.
// Shared by the paint kernels (kernels_painter.cu) and the test oracle of frames over a background.
#pragma once

#define FORMA_SRGB_DECODE_TABLE \\
    {{ \\
""" + " \\\n".join(rows) + " \\\n    }\n"
    with open(OUT, "w") as f:
        f.write(text)
    print(f"wrote {OUT}; bytes off the EOTF's f32: {fixed}")


if __name__ == "__main__":
    sys.exit(main())
