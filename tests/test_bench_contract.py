"""bench.py's JSON contract on the CPU side: the reference arm (`--impl reference`) runs here without a GPU and
must print ONE line with the keys a consumer of the benchmark reads.  It times the unmodified upstream reference, which
is not part of this repository: build() installs it into oracle/_ref/ from a HapHiC checkout (see oracle/refimpl.py)."""

import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_line():
    cmd = [sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1",
           "--contigs", "2000", "--nchr", "4", "--pairs", "1000000", "--cpu-sample-pairs", "200000"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=REPO)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert "unavailable" not in d, d["unavailable"]
    assert d["impl"] == "reference" and d["metric"] == "hic_pairs_per_sec_matrix_build" and d["unit"] == "pairs/s"
    assert d["n_gpus"] == 1 and d["steps"] == 1 and d["warmup"] == 1 and d["higher_is_better"] is True
    assert d["value"] > 0 and d["ms_per_step"] > 0 and d["data"] == "synthetic" and d["vs_baseline"] is None
    assert d["cpu_baseline"]["kind"] == "reference" and d["cpu_baseline"]["cores"] == 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "pairs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and d["mcl"]["unit"] == "iter/s" and d["mcl"]["value"] > 0


def test_reference_arm_other_ranks_stay_silent():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--gpus", "2"],
                       capture_output=True, text=True, timeout=120, cwd=REPO, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""
