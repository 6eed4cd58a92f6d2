"""Runs bench.main() with the DEVICE LAYER STUBBED (no GPU, no libct2b200): a fake `ctranslate2_b200.Generator`, torch.cuda
calls turned into no-ops and gloo in place of nccl.  What is exercised is bench.py's own control flow — the replica line, the
tensor-parallel side record of `--gpus N` and its watchdog — exactly as the driver launches it under torchrun.
STUB_TP_MODE: ok | raise_rank1 (the TP generator of rank 1 fails to build) | hang_rank1 (rank 1 never leaves its decode)."""
import os
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

MODE = os.environ.get("STUB_TP_MODE", "ok")
RANK = int(os.environ.get("RANK", "0"))

torch.cuda.set_device = lambda *a, **k: None
torch.cuda.synchronize = lambda *a, **k: None
torch.cuda.empty_cache = lambda *a, **k: None
_tensor = torch.tensor
torch.tensor = lambda data, device=None, **k: _tensor(data, **k)
_init = dist.init_process_group
dist.init_process_group = lambda backend=None, device_id=None, **k: _init("gloo", **k)


class _Result:
    def __init__(self, n):
        self.sequences_ids = [[0] * n]


class FakeGenerator:
    def __init__(self, model_path, device_index=0, compute_type="default", max_batch_size=32, max_length=0,
                 use_cuda_graph=True, tensor_parallel=False):
        self.tp = tensor_parallel
        if tensor_parallel and MODE == "raise_rank1" and RANK == 1:
            raise RuntimeError("stub: this rank cannot build its shard")

    def info(self):
        return {"weight_bytes": 8037058560}

    def bench_decode(self, batch, prompt_len, steps, warmup):
        if self.tp and MODE == "hang_rank1" and RANK == 1:
            time.sleep(3600)                     # a peer-flag wait that never ends
        return 280.0, (2.7 if self.tp else 3.0) * steps, 292 * steps

    def bench_last_logits(self, batch, vocab_size):
        import numpy as np
        return np.full((batch, vocab_size), 0.5, np.float32)

    def generate_batch(self, prompts, max_length=1, **kw):
        return [_Result(max_length) for _ in range(len(prompts))]

    def close(self):
        pass


fake = types.ModuleType("ctranslate2_b200")
fake.Generator = FakeGenerator
sys.modules["ctranslate2_b200"] = fake

import bench  # noqa: E402

bench.model_dir = lambda *a, **k: "/nonexistent/stub-model"
bench.gemm_roofline = lambda *a, **k: {"bound": "hbm", "achieved": 4477.3, "peak": 6485.2, "unit": "GB/s", "frac": 0.69, "traffic": None}
bench.awq_roofline = bench.gemm_roofline
bench.measure_variant = lambda *a, **k: {"ms_per_step": 3.0, "tokens_per_s": 10000.0}
bench.translate_record = lambda *a, **k: {"decode_ms_per_step": 0.6}
bench.translate_reference = lambda *a, **k: {"ref_cuda": {"tokens_per_s": 1.0}}
bench.ref_cuda_bench = lambda *a, **k: {"decode_tokens_per_s": 1000.0}
bench.reference_cpu = lambda *a, **k: {"value": 12.0, "unit": "tokens/s", "cores": 1, "kind": "reference", "sample": "stub",
                                       "steps": 1, "seconds": 1.0}

if __name__ == "__main__":
    bench.main()
