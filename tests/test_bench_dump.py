"""bench.py --dump-outputs on the GPU: what the timed path computed, written as float64 .npy files."""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_bench_dump_outputs_on_gpu(tmp_path):
    """bench.py --dump-outputs on C1, twice: the same files, float64, within 64 MB, the requested number of timed steps,
    and the same outputs from the same seeded inputs (up to the run-to-run order of the fp64 RED scatter)."""
    import json, subprocess, sys
    dumps = []
    for d in ("a", "b"):
        out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--config", "C1", "--steps", "2", "--warmup", "0",
                              "--no-cpu-baseline", "--no-e2e", "--no-extra-configs", "--dump-outputs", str(tmp_path / d)],
                             capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert out.returncode == 0, out.stderr[-3000:]
        assert json.loads(out.stdout.strip().splitlines()[-1])["steps"] == 2
        files = sorted(os.listdir(tmp_path / d))
        assert files == ["chi2.npy", "point.npy", "pose.npy"], files
        assert sum(os.path.getsize(tmp_path / d / f) for f in files) <= 64 << 20
        dumps.append({f: np.load(tmp_path / d / f) for f in files})
    for f, a in dumps[0].items():
        b = dumps[1][f]
        assert a.dtype == np.float64 and a.shape == b.shape
        assert np.allclose(a, b, rtol=1e-9, atol=1e-12), (f, np.abs(a - b).max())
