"""BASELINE config 4 on real GPUs: the hash-range-sharded prefix index with its native NCCL exchange
(csrc/shard_exchange.cu) must return, on every rank, exactly what a replicated index returns — and the CPU oracle's
answer on a sample — for the device-pointer call, the host-pointer call, an empty batch on one rank, a forced
bucket-overflow round and the whole xllm_ingest_batch pipeline (scripts/sharded_check.py is the per-rank worker,
launched here with torchrun, one process per GPU).  Needs >= 2 GPUs."""
import json
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_equals_replicated_equals_oracle(world):
    if _n_gpus() < world:
        pytest.skip("needs %d GPUs" % world)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "scripts", "sharded_check.py"), "--requests", "4096", "--index-keys",
                        str(1 << 18), "--iters", "3"], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert p.returncode == 0, (p.stdout[-3000:], p.stderr[-3000:])
    line = [ln for ln in p.stdout.split("\n") if ln.startswith("{")][-1]
    out = json.loads(line)
    assert out["n_gpus"] == world and out["check"].startswith("sharded == replicated")
