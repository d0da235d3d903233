"""bench.py's output contract: the reference arm (`--impl reference`, the unmodified src/fsk.c on the host
cores) and the GPU arm each print ONE JSON line with the contract keys; under a multi-rank launch only rank 0
prints."""
import json
import os
import subprocess
import sys

import pytest

import orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_bench(extra_env=None):
    env = dict(os.environ, **(extra_env or {}))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                        "--warmup", "0", "--cpu-streams", "8", "--nsamples", "48000"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, r.stderr[-800:]
    return [ln for ln in r.stdout.decode().splitlines() if ln.strip()]


def test_reference_arm_prints_one_contract_line():
    lines = run_bench()
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference"
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e", "gpu_launches"):
        assert key in d, key
    assert d["metric"].startswith("audio Msamples/s demodulated") and d["unit"] == "Msamples/s"
    assert d["higher_is_better"] is True and d["vs_baseline"] is None and d["gpu_launches"] == 0
    assert "workload" in d["config"] and "model" not in d["config"]
    cb = d["cpu_baseline"]
    assert cb["kind"] == ("reference" if orc.have_ref() else "port") and cb["cores"] >= 1 and cb["value"] > 0
    assert cb["value"] == d["value"] == d["e2e"]["value"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    if orc.have_ref():
        assert "not FFTW" in cb["sample"]           # the stand-in FFT is named, whichever it is


def test_reference_arm_other_ranks_stay_silent():
    assert run_bench({"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2"}) == []


@pytest.fixture(scope="module")
def gpu_line(tmp_path_factory):
    """One `python bench.py` run on the GPU: the headline at a small size with `--steps 2`, every `configs` entry
    at its own size with one timed step, and `--dump-outputs`.  Returns (JSON line, dump directory)."""
    out = tmp_path_factory.mktemp("bench") / "dump"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "2", "--warmup", "3",
                        "--streams", "4096", "--nsamples", "48000", "--e2e-streams", "1024", "--no-cpu",
                        "--config-steps", "1", "--dump-outputs", str(out)],
                       cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1500)
    assert r.returncode == 0, r.stderr[-800:]
    lines = [ln for ln in r.stdout.decode().splitlines() if ln.strip()]
    assert len(lines) == 1
    return json.loads(lines[0]), out


@pytest.mark.gpu
def test_gpu_line_has_the_contract_keys(gpu_line):
    """The headline: the contract keys, one rx launch per timed step (`--steps` sets their number), and
    `--dump-outputs` writing the records of the last step."""
    d, out = gpu_line
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "roofline", "cpu_baseline", "e2e", "gpu_launches", "clocks"):
        assert key in d, key
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] == 3 and d["gpu_launches"] == 2
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0
    assert d["e2e"]["value"] < d["value"]                       # host buffers: PCIe-bound, not a copy of `value`
    assert "workload" in d["config"] and d["dtype"] == "f32" and d["data"] == "synthetic"
    import numpy as np
    import minimodem_b200 as mm
    files = sorted(os.listdir(out))
    assert files == ["frames.npy", "rows.npy", "states.npy"]
    assert sum(os.path.getsize(out / f) for f in files) <= 64_000_000
    st, fr = np.load(out / "states.npy"), np.load(out / "frames.npy")
    assert st.dtype == fr.dtype == np.float64 and st.shape[0] == fr.shape[0] == 4096
    col = {n: i for i, n in enumerate(mm.STATE_DTYPE.names)}
    assert (st[:, col["done"]] == 1).all() and (st[:, col["nframes"]] >= 1).all()


@pytest.mark.gpu
def test_gpu_line_carries_every_baseline_configuration(gpu_line):
    """The `configs` block: every other BASELINE configuration, each with kernel time, roofline fraction, the
    kernel variant that ran and a decode check on >= 1 % of the streams (exact wherever the signal is clean or
    only offset); RTTY and Bell103 on the prefix-table kernel."""
    d, _ = gpu_line
    keys = [c["key"] for c in d["configs"]]
    for want in ("cfg2_1200_awgn", "cfg3_rtty_8k", "cfg4_bell103_offset0.00", "cfg4_bell103_awgn0.50", "cfg5_same_per_gpu"):
        assert any(k.startswith(want) for k in keys), (want, keys)
    for c in d["configs"]:
        assert c["value"] > 0 and 0 < c["roofline_frac"] < 1 and c["kernel_ms"] > 0 and c["kernel"].startswith("k_rx<")
        assert c["decode_check"]["streams"] * 100 >= c["streams_per_gpu"]
        if "awgn0.50" not in c["key"]:
            assert c["decode_check"]["fraction_exact"] == 1.0, c["key"]
    by = {c["key"]: c for c in d["configs"]}
    assert "prefix-table" in by["cfg3_rtty_8k_clean"]["kernel"] and "prefix-table" in by["cfg4_bell103_offset0.00"]["kernel"]
