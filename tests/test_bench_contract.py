"""bench.py's reference arm is CPU-only, so its side of the measurement contract can be checked
without a GPU: ONE JSON line on stdout with the agreed keys."""
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line():
    out = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference",
                          "--batch", "4", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=600, check=True).stdout
    lines = [l for l in out.splitlines() if l.strip()]
    assert len(lines) == 1, out
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "quicknet_images_per_sec"
    assert d["unit"] == "images/s" and d["higher_is_better"] is True and d["value"] > 0
    assert d["n_gpus"] == 1 and d["steps"] == 1 and d["vs_baseline"] is None
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "images/s", "h2d_bytes_per_step": 0,
                        "d2h_bytes_per_step": 0}
