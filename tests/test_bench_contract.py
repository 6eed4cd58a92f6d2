"""bench.py contract, CPU side: the reference arm (`--impl reference`) runs the unmodified reference build under
oracle/_ref on the host cores and prints ONE JSON line with the keys the driver reads.  (The CUDA arm needs a GPU and is
exercised by the driver; its line carries the same keys plus roofline / clocks / gpu_launches.)"""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import refapi  # noqa: E402


@pytest.mark.skipif(not refapi.available(), reason="oracle/_ref not built")
@pytest.mark.timeout(300)
def test_reference_arm_prints_the_contract_line(tmp_path):
    env = dict(os.environ, CT2B200_BENCH_DIR=str(tmp_path))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--model", "tiny", "--batch", "4",
                        "--steps", "2", "--warmup", "1"], capture_output=True, text=True, env=env, timeout=280)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "generate_batch tokens/sec" and d["unit"] == "tokens/s"
    for key in ("value", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
                "data", "config", "cpu_baseline", "e2e"):
        assert key in d, key
    assert d["higher_is_better"] is True and d["value"] > 0 and "workload" in d["config"]
    assert d["cpu_baseline"]["kind"] == "reference" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_step_bytes_matches_survey_figures():
    """SURVEY §8(d): Llama-3-8B INT8 streams 7,504,658,432 weight bytes per decode step + 131,072 B of KV per cached token."""
    import bench
    w = bench.step_bytes("8b", 0, 0)
    assert abs(w - (7504658432 + 4 * (32 * (6144 + 4096 + 2 * 14336 + 4096) + 128256))) == 0
    assert bench.step_bytes("8b", 1, 1) - w == 131072


@pytest.mark.skipif(not refapi.available(), reason="oracle/_ref not built")
@pytest.mark.timeout(400)
def test_reference_arm_under_torchrun_prints_one_line(tmp_path):
    """Launched like the driver launches N > 1 (`python -m torch.distributed.run --nproc-per-node N bench.py --impl reference
    --gpus N ...`): rank 0 alone runs the reference and prints the line, the other ranks exit 0 without work."""
    env = dict(os.environ, CT2B200_BENCH_DIR=str(tmp_path))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29931", os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--model", "tiny",
           "--batch", "2", "--steps", "2", "--warmup", "1"]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=380)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["value"] > 0


def test_tp_watchdog_prints_the_replica_line_and_leaves():
    """`bench.py --gpus N` adds a tensor-parallel side record whose collectives are spin waits inside kernels: a failing rank
    must not cost the driver its line.  The watchdog prints the line rank 0 already holds (failure under `tp.error`) and
    exits 0; a cancelled watchdog does nothing."""
    code = ("import bench, time\n"
            "w = bench.TpWatchdog(0.3, {'metric': 'generate_batch tokens/sec', 'value': 1.0})\n"
            "time.sleep(20)\nprint('not reached')\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=60)
    assert r.returncode == 0, r.stderr
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1 and "not reached" not in r.stdout
    d = json.loads(lines[0])
    assert d["value"] == 1.0 and "timed out" in d["tp"]["error"] and "error" in d["roofline"]
    # ranks other than 0 hold no line: they leave silently
    code = "import bench, time\nw = bench.TpWatchdog(0.3, None)\ntime.sleep(20)\nprint('not reached')\n"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=60)
    assert r.returncode == 0 and r.stdout == ""
    code = "import bench, time\nw = bench.TpWatchdog(0.3, {'a': 1})\nw.cancel()\ntime.sleep(1)\nprint('alive')\n"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=60)
    assert r.stdout.strip() == "alive"


_KEYS = ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
         "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline")


def _run_stub(world, mode="ok", extra=(), port=29941):
    env = dict(os.environ, STUB_TP_MODE=mode)
    worker = os.path.join(ROOT, "tests", "bench_stub_worker.py")
    if world == 1:
        cmd = [sys.executable, worker, "--steps", "8", "--warmup", "3"] + list(extra)
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
               "127.0.0.1", "--master-port", str(port), worker, "--gpus", str(world), "--steps", "8", "--warmup", "3"] + list(extra)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=280)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    return r, lines


@pytest.mark.timeout(300)
def test_own_arm_control_flow_one_gpu_stubbed_device():
    """bench.py's own arm with the device layer stubbed (tests/bench_stub_worker.py): ONE line with every key of the contract,
    the four variants, translate and cpu_baseline records."""
    r, lines = _run_stub(1)
    assert r.returncode == 0, r.stderr[-2000:]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    for k in _KEYS + ("e2e_full", "variants", "translate", "cpu_baseline"):
        assert k in d, k
    assert d["n_gpus"] == 1 and d["scaling"] == "weak" and d["value"] == pytest.approx(32 * 8 / (3.0 * 8 * 1e-3), rel=1e-6)
    assert set(d["variants"]) == {"int8_b1", "int8_b32", "awq_b1", "awq_b32"} and "ref_cuda_flash" in d["variants"]["int8_b32"]
    assert "tp" not in d


@pytest.mark.timeout(300)
def test_own_arm_under_torchrun_world2_gloo_replicas_and_tp_record():
    """`--gpus 2` as the driver launches it (gloo stands in for nccl): rank 0 prints ONE line, value aggregates both replicas
    (weak scaling), and the `tp` record carries the strong-scaling step of one tensor-parallel generator."""
    r, lines = _run_stub(2, port=29942)
    assert r.returncode == 0, r.stderr[-2000:]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    for k in _KEYS:
        assert k in d, k
    assert d["n_gpus"] == 2 and d["scaling"] == "weak" and d["value"] == pytest.approx(2 * 32 * 8 / (3.0 * 8 * 1e-3), rel=1e-6)
    assert d["config"]["global_batch"] == 64
    assert d["tp"]["parallelism"] == "tp2" and d["tp"]["scaling"] == "strong" and d["tp"]["ms_per_step"] == pytest.approx(2.7)
    assert d["tp"]["speedup_vs_one_gpu_step"] == pytest.approx(3.0 / 2.7, abs=1e-3)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("mode", ["raise_rank1", "hang_rank1"])
def test_tp_record_failure_keeps_the_replica_line(mode):
    """A rank that cannot build its tensor-parallel shard, or one that never leaves a peer-flag wait: the driver still gets the
    replica line (exit 0, ONE line) with the failure under `tp.error`."""
    r, lines = _run_stub(2, mode=mode, extra=("--tp-timeout", "6"), port=29943 if mode == "raise_rank1" else 29944)
    assert r.returncode == 0, r.stderr[-2000:]
    assert len(lines) == 1, r.stdout + r.stderr[-1500:]
    d = json.loads(lines[0])
    assert d["n_gpus"] == 2 and d["value"] > 0 and "error" in d["tp"], d.get("tp")


@pytest.mark.timeout(300)
def test_dump_outputs_writes_the_last_step_logits(tmp_path):
    """`--dump-outputs DIR` (device layer stubbed): DIR/logits.npy holds what the last timed step computed, [batch, vocab]
    float32 within 64 MB, beside the unchanged result line; the reference arm refuses the flag instead of ignoring it."""
    import numpy as np
    out = tmp_path / "dump"
    r, lines = _run_stub(1, extra=("--no-variants", "--no-cpu-baseline", "--dump-outputs", str(out)))
    assert r.returncode == 0, r.stderr[-2000:]
    assert len(lines) == 1 and json.loads(lines[0])["steps"] == 8
    assert sorted(os.listdir(out)) == ["logits.npy"]
    a = np.load(out / "logits.npy")
    assert a.dtype == np.float32 and a.shape == (32, 128256) and a.nbytes <= 64 << 20 and (a == 0.5).all()
    r, lines = _run_stub(1, extra=("--impl", "reference", "--dump-outputs", str(tmp_path / "none")))
    assert r.returncode != 0 and not lines and not os.path.exists(tmp_path / "none")
