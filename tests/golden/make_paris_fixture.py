"""Parses the reference's benchmark asset into committed fixtures.

    python tests/golden/make_paris_fixture.py <forma checkout>/assets/svgs/paris-30k.svg

Source: assets/svgs/paris-30k.svg of the reference (BASELINE config 2), parsed
by forma_b200/svg.py (the subset loader restating demo/src/demos/svg.rs).
Outputs:
  tests/data/paris30k_paths.npz — path commands + f32 points as handed to
    PathBuilder (group transform applied), linear fill colours, fill rules.
    bench.py and the tests read this file, so the SVG itself is not needed.
  tests/golden/paris30k_excerpt.svg — the file's group with a sample of its <path>
    elements (excerpt_indices), which tests/test_svg_loader.py parses and compares
    with the same paths of the fixture.
"""
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from forma_b200 import svg  # noqa: E402

OUT = os.path.join(ROOT, "tests", "data", "paris30k_paths.npz")
EXCERPT = os.path.join(ROOT, "tests", "golden", "paris30k_excerpt.svg")


def excerpt_indices(n_paths):
    """Every 1250th path and the last one (kept in step with tests/test_svg_loader.py)."""
    return list(range(0, n_paths - 1, 1250)) + [n_paths - 1]


def write_excerpt(src, out=EXCERPT):
    """Keeps every element of the file but the <path>s that excerpt_indices does not pick, so
    that the picked ones stay inside their groups."""
    text = open(src).read()
    keep = set(excerpt_indices(len(re.findall(r"<path [^>]*/>", text))))
    count = iter(range(len(text)))
    with open(out, "w") as f:
        f.write(re.sub(r"<path [^>]*/>", lambda m: m.group() + "\n" if next(count) in keep else "", text))


if __name__ == "__main__":
    src = sys.argv[1]
    t0 = time.time()
    paths = svg.parse_svg(src)
    paths.save(OUT)
    write_excerpt(src)
    print(f"{len(paths)} paths, {len(paths.cmd)} commands, {len(paths.pts)} points in {time.time() - t0:.1f}s -> {OUT} "
          f"({os.path.getsize(OUT) / 1e6:.1f} MB)")
    import numpy as np
    print("commands:", dict(zip(*np.unique(paths.cmd, return_counts=True))))
    print("opaque layers:", int((paths.color[:, 3] == 1.0).sum()), "bbox:", paths.pts.min(0), paths.pts.max(0))
