"""bench.py's reference arm on CPU (the GPU arm needs an H100): one JSON line on stdout with the contract's keys."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line():
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [l for l in p.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, p.stdout[-2000:]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "agent_events_per_sec" and d["unit"] == "events/s"
    for key in ("value", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "dtype", "data", "config"):
        assert key in d
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["value"] > 0


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    assert p.returncode == 0 and p.stdout.strip() == "", (p.stdout[-500:], p.stderr[-500:])


def test_dump_outputs_writes_float_arrays_under_64_mb(tmp_path):
    """--dump-outputs on a stand-in engine whose tables exceed the caps: float32/float64 .npy files, seeded samples
    (the same on a second call), CRC-32 and length of the engine's payloads, 64 MB at most"""
    import zlib
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    from calfkit.engine._lib import COL, NUM_COLS, PUB_DTYPE

    class Eng:
        def __init__(self, n):
            rng = np.random.default_rng(1)
            self.ln = rng.integers(0, 64, n).astype(np.uint32)
            self.ln[::256] = 1500                               # longer than the 1 KB head kept of a sampled payload
            self.off = np.zeros(n + 1, np.int64)
            self.off[1:] = np.cumsum(self.ln)
            self.out = rng.integers(0, 256, int(self.off[-1])).astype(np.uint8)
            self.pubs = np.zeros(2 * n, PUB_DTYPE)
            self.pubs["payload"] = np.repeat(np.arange(n), 2)
            self.cols = np.zeros((NUM_COLS, n), np.uint32)
            self.cols[COL["STATUS"]] = np.arange(n) % 7

        def _fetch(self):
            return self.out, self.off, self.ln, self.pubs

        def columns(self):
            return self.cols

    eng = Eng(1_200_000)
    a, b = tmp_path / "a", tmp_path / "b"
    bench.dump_outputs(eng, str(a))
    bench.dump_outputs(eng, str(b))
    files = sorted(p.name for p in a.iterdir())
    assert files == sorted(p.name for p in b.iterdir())
    assert sum((a / f).stat().st_size for f in files) <= 64 << 20
    arrs = {f[:-4]: np.load(a / f) for f in files}
    for f in files:
        assert arrs[f[:-4]].dtype in (np.float32, np.float64)
        assert np.array_equal(arrs[f[:-4]], np.load(b / f))
    pi = arrs["payload_index"].astype(np.int64)
    assert len(pi) == 1 << 20 and np.array_equal(arrs["payload_len"], eng.ln[pi].astype(np.float32))
    for j in (0, 1, len(pi) // 2, len(pi) - 1):
        i = pi[j]
        assert arrs["payload_crc32"][j] == zlib.crc32(eng.out[eng.off[i]:eng.off[i] + eng.ln[i]].tobytes())
    head = arrs["payload_sample_head"]
    for j, i in enumerate(arrs["payload_sample_index"].astype(np.int64)):
        k = min(int(eng.ln[i]), 1024)
        assert np.array_equal(head[j, :k], eng.out[eng.off[i]:eng.off[i] + k]) and (head[j, k:] == -1).all()
    ri = arrs["record_index"].astype(np.int64)
    assert np.array_equal(arrs["record_status"], (ri % 7).astype(np.float32))
    qi = arrs["publishes_index"].astype(np.int64)
    assert np.array_equal(arrs["publishes"][:, 0], (qi // 2).astype(np.float64))
