"""CPU: the byte model behind bench.py's roofline numbers reproduces BASELINE.md section 3 / SURVEY.md section 8d."""
import importlib.util
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bench)


def test_step_bytes_match_baseline_table():
    N, E, T, d = 1920, 23040, 276480, 256
    fwd_inf = lambda nn, ne: 4 * d * (2 * nn + 2 * ne) + 8 * ne     # noqa: E731  (BASELINE.md: 51.30 MB / 615.63 MB)
    assert round(fwd_inf(N, E) / 1e6, 2) == 51.30
    assert round(fwd_inf(E, T) / 1e6, 2) == 615.63
    assert round((4 * (fwd_inf(N, E) + fwd_inf(E, T)) + 4 * fwd_inf(N, E)) / 1e9, 3) == 2.873
    total = bench.step_bytes(N, E, T, d, 4, 4)
    assert round(total / 1e9, 2) == 10.04                             # 156.9 MB per graph at batch 64
    assert round(total / 64 / 1e6, 1) == 156.9


def test_peak_source_is_the_measured_file_when_present():
    peak, src = bench.peaks()
    if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")):
        assert src.startswith("measured") and 3000 < peak < 9000
    else:
        assert src.startswith("fallback") and peak == 3350.0               # H100 SXM data-sheet HBM3 bandwidth
