"""CPU checks of bench.py's bookkeeping (no GPU): the step sizing, the config both arms print, and the ncu-traffic stamp."""
import importlib.util
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bench)


def test_a_step_is_at_least_two_thousand_passes_in_total():
    for steps in (1, 3, 20, 100, 2000, 5000):
        r = bench.passes_per_step(steps)
        assert r >= 1 and r * steps >= 2000 and (r - 1) * steps < 2000 or r == 1       # >= ~2.5 s at 1.3 ms per pass
    assert bench.passes_per_step(20, override=7) == 7


def test_both_arms_print_the_same_config():
    a = bench.bench_config(8, bench.passes_per_step(20))
    b = bench.bench_config(8, bench.passes_per_step(20), P_mean=1.0)                    # the b200 arm adds measured extras
    assert a["workload"] == b["workload"] == bench.WORKLOAD
    assert all(a[k] == b[k] for k in ("views_per_pass_per_gpu", "passes_per_step", "views_per_step_per_gpu"))
    assert a["views_per_step_per_gpu"] == 8 * 100 and "model" not in a


def test_traffic_stamp_matches_code_not_comments(tmp_path, monkeypatch):
    h = bench._source_hash("render_forward_kernel")
    assert re.fullmatch(r"[0-9a-f]{64}", h) and h != bench._source_hash("render_backward_q_kernel")
    # a capture file with one entry stamped with the current code and one stamped with other code
    j = {"render_forward_kernel": {"source_sha256": h, "dram_bytes_per_launch": 5.0e7},
         "render_backward_q_kernel": {"source_sha256": "0" * 64, "dram_bytes_per_launch": 9.0e7}}
    tf = tmp_path / "render_forward_traffic.json"
    tf.write_text(json.dumps(j))
    monkeypatch.setattr(bench, "TRAFFIC_FILE", str(tf))
    val, src = bench._traffic("render_forward_kernel")
    assert val == j["render_forward_kernel"]["dram_bytes_per_launch"]                  # stamp matches the code: reported
    val, src = bench._traffic("render_backward_q_kernel")                               # kernel code changed since the capture:
    assert val is None and src.startswith("stale")                                      # refused, never silently reported
    assert bench._traffic("no_such_kernel")[0] is None
    monkeypatch.setattr(bench, "TRAFFIC_FILE", str(tmp_path / "absent.json"))
    assert bench._traffic("render_forward_kernel")[0] is None                           # no capture: nothing reported
