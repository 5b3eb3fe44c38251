"""CPU checks of bench.py's own pieces: the synthetic window generator of the roofline_hbm block (SURVEY 8d: distinct,
sorted genes), the counting adjacency that lets the UNMODIFIED generate_pathSet be timed on a bounded sample, and the
--dump-outputs writer."""
import os
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import bench  # noqa: E402
from oracle import ref_import  # noqa: E402


def test_synthetic_windows_are_sorted_distinct_and_reproducible():
    import torch
    rowptr, gene, label = bench.synthetic_windows(500, 3000, 80, torch.device("cpu"), seed=777)
    g = gene.view(500, 80).numpy()
    assert (np.diff(g, axis=1) > 0).all() and g.min() >= 0 and g.max() < 3000       # strictly ascending = distinct
    assert rowptr.tolist() == list(range(0, 501 * 80, 80)) and set(label.tolist()) <= {0, 1}
    r2, g2, l2 = bench.synthetic_windows(500, 3000, 80, torch.device("cpu"), seed=777)
    assert (g2 == gene).all() and (l2 == label).all()
    assert 0.3 < float(label.float().mean()) < 0.7


def test_counting_adjacency_counts_visits_and_stops_on_budget():
    from tests import helpers
    rp, col, w = helpers.random_graph(200, 6, seed=3)
    A = bench.CountingAdjacency(rp, col, w, budget_s=0.2)
    row = A[5]
    assert row.shape == (200,) and row.dtype == np.float32 and A.visits == 1
    assert (np.nonzero(row)[0] == col[rp[5]:rp[6]]).all()
    time.sleep(0.25)
    with pytest.raises(bench.CountingAdjacency.TimeUp):
        A[6]


@pytest.mark.skipif(not ref_import.available(), reason="reference script not staged")
def test_reference_walk_is_timed_through_its_own_function():
    from tests import helpers
    ref = ref_import.load()
    rp, col, w = helpers.random_graph(150, 5, seed=4)
    rate, visits, dt = bench.cpu_walk_rate(ref, [(rp, col, w)], 20, 0.5, 1)
    assert visits > 200 and 0.4 < dt < 5 and rate == pytest.approx(visits / dt)


def test_dump_outputs_writes_exact_float_arrays_and_a_fixed_sample(tmp_path):
    ids = bench.dump_sample(100_000, 4096)
    assert len(ids) == 4096 and (np.diff(ids) > 0).all() and (ids == bench.dump_sample(100_000, 4096)).all()
    assert (bench.dump_sample(10, 4096) == np.arange(10)).all()
    rows = np.arange(2**31 - 64, 2**31 - 1, dtype=np.int32).reshape(3, 21)
    bench.dump_outputs(str(tmp_path / "out"), {"rows": rows, "w": np.linspace(0, 1, 7, dtype=np.float64)})
    got = np.load(tmp_path / "out" / "rows.npy")
    assert got.dtype == np.float64 and (got == rows).all()
    assert np.load(tmp_path / "out" / "w.npy").dtype == np.float32
    with pytest.raises(AssertionError):
        bench.dump_outputs(str(tmp_path / "big"), {"x": np.zeros((65 << 20) // 4, np.float32)})
