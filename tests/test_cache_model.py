"""The oracle's layer cache held to the NumPy model of tests/cache_model.py on every named edit sequence
of tests/cache_sequences.py: frame by frame, the model's frame (the bytes before the frame, with the
tiles it decides to write taken from an uncached frame) equals the oracle's byte for byte, and every
sequence reaches the tile decisions it is named for. Three planted model errors must each be caught.
tests/test_gpu_cache_limits.py then holds the device to the same frames and write sets."""
import numpy as np
import pytest

import cache_model
import cache_sequences as cq


@pytest.fixture(scope="module")
def recorded(oracle_api):
    runs = {}

    def get(name):
        if name not in runs:
            runs[name] = cq.run(name, oracle_api, record=True)
        return runs[name]
    return get


def replay(s, errors=()):
    """The model's frames and ops of a recorded session."""
    m = cache_model.CacheModel(errors)
    return [m.frame(f, before) for f, (before, _) in zip(s.inputs, s.frames)]


def first_difference(s, errors=()):
    for k, ((want, ops), (_, got)) in enumerate(zip(replay(s, errors), s.frames)):
        bad = np.argwhere((want != got).any(axis=2))
        if len(bad):
            y, x = bad[0].tolist()
            return (f"frame {k}: {len(bad)} pixels differ, first (x {x}, y {y}): model {want[y, x].tolist()} "
                    f"({ops.get((x // 16, y // 16))}), oracle {got[y, x].tolist()}")
    return None


def in_range(n, want):
    lo, hi = want if isinstance(want, tuple) else (want, want)
    return n >= lo and (hi is None or n <= hi)


@pytest.mark.parametrize("name", sorted(cq.SEQUENCES))
def test_model_equals_oracle(recorded, name):
    s = recorded(name)
    assert len(s.inputs) == len(s.frames) > 0
    diff = first_difference(s)
    assert diff is None, diff


@pytest.mark.parametrize("name", sorted(cq.SEQUENCES))
def test_sequence_reaches_its_condition(recorded, name):
    s = recorded(name)
    frames = replay(s)
    for k, want in s.wants:
        ops = frames[k][1]
        for op, n in want.items():
            got = cache_model.count(ops, op) if op != "written" else \
                cache_model.count(ops, cache_model.SOLID) + cache_model.count(ops, cache_model.PAINT)
            assert in_range(got, n), f"frame {k}: {got} tiles {op}, the sequence wants {n}"


# Each planted error, and a sequence that catches it.
PLANTED = [("removed", "decision_edges"), ("unmapped", "frame_state"), ("clear", "frame_state")]


@pytest.mark.parametrize("error,name", PLANTED)
def test_planted_model_error_is_caught(recorded, error, name):
    assert first_difference(recorded(name), (error,)) is not None, f"the model with error {error!r} still equals the oracle"
