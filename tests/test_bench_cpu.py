"""bench.py's stdout contract, as far as a machine without a GPU can check it: the result is ONE JSON line on the
process's stdout, whatever libraries write to file descriptor 1 (NCCL's version banner did), and the reference arm
(the oracle port on the host cores) produces the line the driver expects."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_result_line_is_alone_on_stdout():
    code = ("import os, bench\n"
            "bench.claim_stdout()\n"
            "os.write(1, b'NCCL version 0.0.0\\n')\n"      # a library writing to fd 1 behind Python's back
            "print('chatter')\n"
            "bench.emit({'metric': 'm', 'value': 1.5})\n")
    p = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr
    assert json.loads(p.stdout) == {"metric": "m", "value": 1.5}       # exactly one line, and it parses
    assert "NCCL version" in p.stderr and "chatter" in p.stderr


def test_reference_arm_line():
    env = dict(os.environ, RANK="0", WORLD_SIZE="1")
    p = subprocess.run([sys.executable, "bench.py", "--impl", "reference", "--steps", "1", "--warmup", "0", "--scale", "0.02"],
                       cwd=ROOT, capture_output=True, text=True, timeout=600, env=env)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = p.stdout.strip().splitlines()
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["higher_is_better"] is True
    assert d["metric"] == "haystack_GB_per_s_scanned_find_matches_as_indexes" and d["unit"] == "GB/s" and d["value"] > 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_dump_outputs_float64_within_budget(tmp_path):
    """--dump-outputs: float64 arrays; above the budget, the same seeded sample of rows every time."""
    import numpy as np
    import torch

    import bench

    rows = np.arange(4 * 5000, dtype=np.uint32).reshape(5000, 4)
    rows[:, 3] = 0xFFFFFFF0   # uint32 values above 2^31 survive the int32 view the scan returns
    m = torch.from_numpy(rows.view(np.int32))
    mo = torch.arange(101, dtype=torch.int64) * 50
    bench.dump_outputs(str(tmp_path / "a"), m, mo, 5000, budget=1 << 30)
    got = np.load(tmp_path / "a" / "matches.npy")
    assert got.dtype == np.float64 and np.array_equal(got, rows.astype(np.float64))
    assert np.array_equal(np.load(tmp_path / "a" / "match_offsets.npy"), mo.numpy().astype(np.float64))
    assert np.load(tmp_path / "a" / "total.npy").tolist() == [5000.0]
    for d in ("b", "c"):
        bench.dump_outputs(str(tmp_path / d), m, mo, 5000, budget=64 << 10)
    files = sorted(os.listdir(tmp_path / "b"))
    assert files == ["match_offsets.npy", "matches.npy", "matches_index.npy", "total.npy"]
    assert sum(os.path.getsize(tmp_path / "b" / f) for f in files) <= 64 << 10
    idx = np.load(tmp_path / "b" / "matches_index.npy").astype(np.int64)
    assert np.array_equal(np.load(tmp_path / "b" / "matches.npy"), rows[idx].astype(np.float64))
    for f in files:
        assert np.array_equal(np.load(tmp_path / "b" / f), np.load(tmp_path / "c" / f))


def test_reference_arm_other_ranks_stay_silent():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    p = subprocess.run([sys.executable, "bench.py", "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0"],
                       cwd=ROOT, capture_output=True, text=True, timeout=120, env=env)
    assert p.returncode == 0 and p.stdout.strip() == ""
