"""NumPy replay of the indexing flatten_eval_kernel does (forma_b200/csrc/kernels_raster.cu), a
check of its quad choice against the reference's quad walk, and the pre-flight budget every
scene passes before the device sees it.

`replay(batch)` follows one thread per output point through the records of a batch laid out the
way `Renderer::flush_geometry` stages it (`layout`): the job bisection, then either the point
record or the spline bisection and the quad bisection of the spline. For every point it gives
the kind (0 literal, 1 literal that ends a contour, 2 evaluated at pi, 3 evaluated with a recorded
numerator), the record it reads, the quad it evaluates, pi, the contour flag and the geometry
id, and it asserts every index the kernel forms is inside its array, as well as the invariants
those indices rest on: a spline with evaluated points has at least one quad, a point record's
quad lies inside its own job's quads, `quad_base + first_quad + a` stays in the batch, and the
running curvatures the kernel bisects are sorted within each spline.

`reference_walk_mismatch(batch, replayed)` computes the reference's quad walk from the same
records (path.rs:424-431, restated in oracle/path.hpp `into_segments`): one quad index `i` per
path, `if pi > total[i] { i += 1 }` per evaluated point, and `i += 1` after every spline with
subdivisions. Both sides only compare float32 values with `(float)pi`, so the model is exact;
the float arithmetic of the evaluation is left to the device comparisons.

`preflight(...)` is the budget: the program's point count (program_stats) and the oracle's
pixel-segment count (rasterize_only) under caps, and no line that survives the skip rules with a
non-finite end point. Such a line gets a saturated length of 0xFFFFFFFF on the device, and a sum
of such lengths wraps the u32 block totals of line_count_kernel / raster_emit_kernel (DESIGN.md §5).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from forma_b200.binding import POINT_REC, QUAD_REC, SPLINE_REC

EVAL_MASK = (1 << 30) - 1
POINT_CAP = 20_000_000     # points a device scene may have (flattened: 12 B each on the device)
SEGMENT_CAP = 50_000_000   # pixel segments a rendered scene may have (8 B each, sorted twice)


class ModelError(AssertionError):
    pass


def _check(cond, what):
    if not bool(np.all(cond)):
        raise ModelError(what)


@dataclass
class Batch:
    """What flush_geometry uploads for one batch of inserts (device_types.h FlattenJob)."""
    first_point: np.ndarray  # u32 per job
    quad_base: np.ndarray
    spline_base: np.ndarray
    n_splines: np.ndarray
    geom_id: np.ndarray
    xf_index: np.ndarray
    splines: np.ndarray      # SPLINE_REC
    points: np.ndarray       # POINT_REC
    kinds: np.ndarray        # u8
    quads: np.ndarray        # QUAD_REC
    n_points: int

    @property
    def n_jobs(self) -> int:
        return len(self.first_point)


def layout(programs: Sequence[dict], geom_ids: Optional[Sequence[int]] = None,
           has_xf: Optional[Sequence[bool]] = None) -> Batch:
    """Stages the programs (Path.program()) of consecutive inserts like flush_geometry: job j
    starts at the sum of the earlier jobs' points, quads, spline records or point records."""
    n = len(programs)
    geom_ids = list(geom_ids) if geom_ids is not None else list(range(1, n + 1))
    has_xf = list(has_xf) if has_xf is not None else [False] * n
    cols = {k: np.zeros(n, np.uint32) for k in ("first_point", "quad_base", "spline_base", "n_splines", "geom_id",
                                                  "xf_index")}
    pi = qi = si = ri = xi = 0
    for j, p in enumerate(programs):
        cols["first_point"][j] = pi
        cols["quad_base"][j] = qi
        cols["spline_base"][j] = si if len(p["splines"]) else ri
        cols["n_splines"][j] = len(p["splines"])
        cols["geom_id"][j] = geom_ids[j]
        if has_xf[j]:
            xi += 1
            cols["xf_index"][j] = xi
        si += len(p["splines"])
        ri += len(p["points"])
        qi += len(p["quads"])
        pi += p["stats"]["points"]
    cat = lambda key, dt: np.concatenate([p[key] for p in programs]) if programs else np.zeros(0, dt)  # noqa: E731
    return Batch(splines=cat("splines", SPLINE_REC), points=cat("points", POINT_REC), kinds=cat("kinds", np.uint8),
                 quads=cat("quads", QUAD_REC), n_points=pi, **cols)


def _bits(v):
    return np.ascontiguousarray(v, np.float32).view(np.uint32).astype(np.uint64)


def replay(b: Batch) -> dict:
    """Per output point of the batch: job, kind, rec (point record, or spline record, in the
    batch), quad (in the batch; -1 for literals), pi, contour, gid. Raises ModelError when the
    kernel would form an index outside its array or rely on a broken invariant."""
    n = b.n_points
    out = {"job": np.zeros(n, np.int64), "kind": np.zeros(n, np.uint8), "rec": np.zeros(n, np.int64),
           "quad": np.full(n, -1, np.int64), "pi": np.zeros(n, np.float32), "contour": np.zeros(n, bool),
           "gid": np.zeros(n, np.uint32)}
    if n == 0:
        return out
    _check(b.n_jobs > 0, "points without a job")
    fp = b.first_point.astype(np.int64)
    _check(fp[0] == 0, "the first job does not start at point 0")
    _check(np.diff(fp) >= 0, "job first points are not sorted (the job bisection needs them sorted)")
    _check(fp[-1] <= n, "a job starts past the batch's points")
    n_quads_batch = len(b.quads)
    quad_end = np.append(b.quad_base[1:].astype(np.int64), n_quads_batch)
    _check(quad_end >= b.quad_base, "quad bases are not sorted")
    _check(quad_end <= n_quads_batch, "a job's quads run past the batch")
    totals = b.quads["total"] if n_quads_batch else np.zeros(0, np.float32)
    point_a = b.points["a"].view(np.uint32) if len(b.points) else np.zeros(0, np.uint32)
    for j in range(b.n_jobs):
        lo, hi = int(fp[j]), int(fp[j + 1]) if j + 1 < b.n_jobs else n
        if hi == lo:
            continue
        local = np.arange(hi - lo, dtype=np.int64)
        qb, nq_job = int(b.quad_base[j]), int(quad_end[j] - b.quad_base[j])
        kind = np.zeros(hi - lo, np.uint8)
        quad = np.full(hi - lo, -1, np.int64)
        pi = np.zeros(hi - lo, np.float32)
        if b.n_splines[j] == 0:  # point encoding
            rec = int(b.spline_base[j]) + local
            _check(rec[-1] < len(b.points), f"job {j}: point record {rec[-1]} past the batch's {len(b.points)}")
            kind = b.kinds[rec]
            _check(kind <= 3, f"job {j}: unknown point kind")
            ev = kind >= 2
            a = point_a[rec[ev]].astype(np.int64)
            _check(a < nq_job, f"job {j}: a point record's quad lies outside its job's {nq_job} quads")
            quad[ev] = qb + a
            pi[ev] = b.points["b"][rec[ev]]
        else:  # spline encoding
            s0, ns = int(b.spline_base[j]), int(b.n_splines[j])
            _check(s0 + ns <= len(b.splines), f"job {j}: spline records past the batch")
            sp = b.splines[s0:s0 + ns]
            sfp = sp["first_point"].astype(np.int64)
            _check(sfp[0] == 0, f"job {j}: the first spline does not start at point 0")
            _check(np.diff(sfp) >= 0, f"job {j}: spline first points are not sorted")
            s = np.searchsorted(sfp, local, side="right") - 1  # last spline with first_point <= local
            rec = s0 + s
            info = sp["info"].astype(np.int64)
            has_start, evaluated, ends = (info >> 30) & 1, info & EVAL_MASK, (info >> 31) & 1
            width = has_start + evaluated + 1
            _check(sfp[1:] == sfp[:-1] + width[:-1], f"job {j}: a spline's points overlap the next spline's")
            _check(sfp[-1] + width[-1] == hi - lo, f"job {j}: the last spline does not end at the job's last point")
            jj = local - sfp[s]
            hs, ev_n = has_start[s], evaluated[s]
            start = (hs == 1) & (jj == 0)
            end = ~start & (jj - hs == ev_n)
            ev = ~start & ~end
            kind = np.where(end & (ends[s] == 1), 1, 0).astype(np.uint8)
            kind[ev] = 2
            pi[ev] = (jj[ev] - hs[ev] + 1).astype(np.float32)
            if ev.any():
                fq, nqs = sp["first_quad"].astype(np.int64), sp["n_quads"].astype(np.int64)
                used = np.unique(s[ev])
                _check(nqs[used] >= 1, f"job {j}: a spline with evaluated points has no quad")
                _check(fq[used] + nqs[used] <= nq_job, f"job {j}: a spline's quads lie outside its job's quads")
                _check(fq[used][1:] >= fq[used][:-1] + nqs[used][:-1], f"job {j}: splines share quads")
                # sorted running curvatures within each spline; then the bisection's answer is the
                # first quad whose total reaches pi, clamped to the spline's last quad
                spl_of_quad = np.full(nq_job, -1, np.int64)
                for k in used:
                    spl_of_quad[fq[k]:fq[k] + nqs[k]] = k
                jt = totals[qb:qb + nq_job]
                key = (np.where(spl_of_quad >= 0, spl_of_quad, 0).astype(np.uint64) << np.uint64(32)) | _bits(jt)
                inside = spl_of_quad >= 0
                same = inside[1:] & inside[:-1] & (spl_of_quad[1:] == spl_of_quad[:-1])
                _check(~same | (jt[1:] >= jt[:-1]), f"job {j}: running curvatures decrease within a spline")
                # keys of the quads of the used splines are ascending: search them
                qidx = np.nonzero(inside)[0]
                keys = key[qidx]
                want = (s[ev].astype(np.uint64) << np.uint64(32)) | _bits(pi[ev])
                pos = np.searchsorted(keys, want, side="left")
                first_pos = np.searchsorted(qidx, fq[s[ev]])
                a = np.minimum(pos - first_pos, nqs[s[ev]] - 1)
                quad[ev] = qb + fq[s[ev]] + a
        _check(quad < n_quads_batch, f"job {j}: quad index past the batch")
        out["job"][lo:hi] = j
        out["kind"][lo:hi] = kind
        out["rec"][lo:hi] = rec
        out["quad"][lo:hi] = quad
        out["pi"][lo:hi] = pi
        out["contour"][lo:hi] = kind == 1
        none = (kind == 1) | (local + 1 == hi - lo)
        out["gid"][lo:hi] = np.where(none, 0, b.geom_id[j])
    return out


@dataclass
class Mismatch:
    job: int
    point: int     # in the batch
    kernel: int    # quad the kernel evaluates (job-relative)
    walk: int      # quad the reference's walk evaluates (job-relative; may be past the job's quads)

    def __str__(self):
        return f"job {self.job}, point {self.point}: kernel evaluates quad {self.kernel}, the reference's walk quad {self.walk}"


def reference_walk_mismatch(b: Batch, r: dict) -> Optional[Mismatch]:
    """First evaluated point whose quad differs from the reference's walk, or None.

    The walk of a path starts at i = 0; at each evaluated point `if pi > total[i] { i += 1 }`;
    after each spline with subdivisions `i += 1`. Every spline with subdivisions has evaluated
    points (its curvature exceeds 1), and its evaluated points form one run between literal
    points, so the runs of evaluated points stand for those splines. pi is the position in the run
    (1, 2, ...), for kind 3 records too. Assuming the walk agreed so far, it picks at point p
    `prev + (pi > total[prev])`, where prev is the previous point's quad, or one past the quad of
    the previous run's last point at the start of a run."""
    totals = b.quads["total"] if len(b.quads) else np.zeros(0, np.float32)
    for j in range(b.n_jobs):
        sel = np.nonzero((r["job"] == j) & (r["kind"] >= 2))[0]
        if sel.size == 0:
            continue
        qb = int(b.quad_base[j])
        nq = (int(b.quad_base[j + 1]) if j + 1 < b.n_jobs else len(b.quads)) - qb
        k = r["quad"][sel] - qb
        run_start = np.ones(sel.size, bool)
        run_start[1:] = sel[1:] != sel[:-1] + 1
        run_id = np.cumsum(run_start) - 1
        starts = np.nonzero(run_start)[0]
        pos = np.arange(sel.size) - starts[run_id]
        pi = (pos + 1).astype(np.float32)
        prev = np.empty(sel.size, np.int64)
        prev[1:] = k[:-1]
        prev[0] = 0
        later = starts[1:]
        prev[later] = k[later - 1] + 1
        kind2 = r["kind"][sel] == 2
        _check(r["pi"][sel][kind2] == pi[kind2], f"job {j}: a kind-2 point's pi is not its place in its spline")
        ok_prev = prev < nq
        walk = prev.copy()
        tp = np.zeros(sel.size, np.float32)
        tp[ok_prev] = totals[qb + prev[ok_prev]]
        walk[ok_prev] += pi[ok_prev] > tp[ok_prev]
        bad = np.nonzero(~ok_prev | (walk != k))[0]
        if bad.size:
            p = int(bad[0])
            return Mismatch(j, int(sel[p]), int(k[p]), int(walk[p]))
    return None


def check_program(prog: dict) -> dict:
    """Replays one path's program as a batch of one job; returns the replay plus its first
    walk mismatch under "mismatch"."""
    b = layout([prog])
    r = replay(b)
    r["mismatch"] = reference_walk_mismatch(b, r)
    return r


@dataclass
class Budget:
    points: int
    segments: Optional[int]
    nonfinite_lines: int

    def problems(self, point_cap=POINT_CAP, segment_cap=SEGMENT_CAP) -> List[str]:
        out = []
        if self.points > point_cap:
            out.append(f"{self.points} points > {point_cap}")
        if self.segments is not None and self.segments > segment_cap:
            out.append(f"{self.segments} pixel segments > {segment_cap}")
        if self.nonfinite_lines:
            out.append(f"{self.nonfinite_lines} lines survive the skip rules with a non-finite end point")
        return out


def preflight(points: int, oracle_renderer=None, oracle_comp=None, width: int = 0, height: int = 0) -> Budget:
    """Budget of a scene: `points` from program_stats() of its inserts; with an oracle
    composition, the pixel segments of rasterize_only and the lines that survive the skip rules
    (length > 0 in the oracle's line records) with a non-finite end point."""
    if oracle_comp is None:
        return Budget(points, None, 0)
    segs = oracle_renderer.rasterize_only(oracle_comp, width, height)
    lines = oracle_renderer.lines()
    live = lines["lengths"] > 0
    ends = np.stack([lines["x0"], lines["y0"], lines["x0"] + lines["dx"], lines["y0"] + lines["dy"]])[:, live]
    return Budget(points, int(segs.size), int((~np.isfinite(ends)).any(axis=0).sum()))


def assert_preflight(budget: Budget, what: str, **caps) -> None:
    problems = budget.problems(**caps)
    if problems:
        raise AssertionError(f"{what} fails its pre-flight budget: " + "; ".join(problems))
