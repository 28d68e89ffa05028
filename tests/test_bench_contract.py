"""bench.py contract pieces that can be checked without a GPU."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def test_algorithmic_bytes_follows_the_survey_formula():
    # SURVEY.md §8d: cmps*(d*sizeof(T)+8) + hops*(max_degree+1)*4 + d*sizeof(T) + k*8 per query
    c2 = bench.WORKLOADS["c2_1Mx128_f32_l2"]
    assert bench.unit_bytes(c2) == 520
    assert bench.algorithmic_bytes(c2, 3000, 210, 2, 83) == 3000 * 520 + 210 * 336 + 2 * (512 + 80)
    assert bench.unit_bytes(bench.WORKLOADS["c3_1Mx768_f16_ip"]) == 1544
    c4 = bench.WORKLOADS["c4_10Mx128_i8_pq32"]
    assert bench.unit_bytes(c4) == 40  # 32 code bytes + id + output
    # PQ traversal + rerank: L full-precision rows (136 B each) per query on top
    assert bench.algorithmic_bytes(c4, 1000, 100, 1, 83, rerank_rows=100) == 1000 * 40 + 100 * 336 + (128 + 80) + 100 * 136
    assert bench.unit_bytes(bench.WORKLOADS["c5_40Mx96_f32_l2"]) == 392


def test_host_cores_respects_affinity():
    hc = bench.host_cores()
    assert 1 <= hc["threads"] <= hc["cores_affinity"] <= hc["cores_hw"]


def test_data_generators():
    cfg = dict(bench.WORKLOADS["c3_1Mx768_f16_ip"], centers=8)
    x = bench.make_data(cfg, 1, 100, bench.make_centers(cfg))
    assert x.dtype == np.float16 and abs(float((x.astype(np.float32) ** 2).sum(1).mean()) - 1.0) < 1e-2
    cfg = dict(bench.WORKLOADS["c4_10Mx128_i8_pq32"], centers=8)
    y = bench.make_data(cfg, 1, 100, bench.make_centers(cfg))
    assert y.dtype == np.int8 and y.min() >= -127 and np.abs(y).max() > 40
    assert np.array_equal(bench.find_medoid(y), y[np.argmin(((y.astype(np.float32) - y.astype(np.float32).mean(0)) ** 2).sum(1))])


def test_max_degree_is_the_reference_slack():
    assert bench.max_degree(64) == 83 and bench.max_degree(32) == 41  # config/mod.rs:269-275


def test_stdout_carries_exactly_one_json_line():
    """Anything a library writes to file descriptor 1 after start-up must not reach stdout."""
    code = ("import os, sys; sys.path.insert(0, %r); import bench; bench.claim_stdout(); "
            "os.write(1, b'library banner\\n'); print('python noise'); bench.emit({'ok': 1})" % ROOT)
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0
    assert p.stdout.strip().splitlines() == ['{"ok": 1}']
    assert "library banner" in p.stderr and "python noise" in p.stderr


def test_reference_arm_prints_one_json_line_without_a_gpu():
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1",
                        "--workload", "small_100Kx128_f32_l2"], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert p.returncode == 0
    lines = p.stdout.strip().splitlines()
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference"


def test_traffic_json_is_keyed_by_workload(tmp_path, monkeypatch):
    """roofline.traffic comes from an ncu capture of the workload's own search kernel stored as profiles/traffic.json."""
    (tmp_path / "profiles").mkdir()
    monkeypatch.setattr(bench, "ROOT", str(tmp_path))
    assert bench.ncu_traffic("c2_1Mx128_f32_l2") is None  # no capture stored
    t = {"c2_1Mx128_f32_l2": {"search_kernel_dram_bytes_per_launch": 5.0e9},
         "c4_10Mx128_i8_pq32": {"search_kernel_dram_bytes_per_launch": 2.0e9}}
    (tmp_path / "profiles" / "traffic.json").write_text(json.dumps(t))
    assert bench.ncu_traffic("c2_1Mx128_f32_l2") == 5.0e9 and bench.ncu_traffic("c4_10Mx128_i8_pq32") == 2.0e9
    assert bench.ncu_traffic("c3_1Mx768_f16_ip") is None  # no capture under that key
    # round-1 layout (one entry, no key) still reads as the C2 kernel
    (tmp_path / "profiles" / "traffic.json").write_text(json.dumps({"search_kernel_dram_bytes_per_launch": 7.0}))
    assert bench.ncu_traffic("c2_1Mx128_f32_l2") == 7.0 and bench.ncu_traffic("c4_10Mx128_i8_pq32") is None


def test_dump_outputs_writes_float_arrays(tmp_path):
    """--dump-outputs: one .npy per returned array, float32 kept, integer results widened exactly to float64."""
    ids = np.array([[3, 1], [-1, 7]], np.int32)
    dists = np.array([[0.5, 1.25], [np.inf, 2.0]], np.float32)
    bench.dump_outputs(str(tmp_path / "out"), {"ids": ids, "dists": dists})
    got_ids, got_d = np.load(tmp_path / "out" / "ids.npy"), np.load(tmp_path / "out" / "dists.npy")
    assert got_ids.dtype == np.float64 and np.array_equal(got_ids, ids)
    assert got_d.dtype == np.float32 and np.array_equal(got_d, dists)
