"""world_size-3 gloo run of gather_path_rows (the per-asset finals of a sharded joint Monte-Carlo run)."""
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]

WORKER = r'''
import os, sys
sys.path.insert(0, os.environ["B200BT_ROOT"])
import torch, torch.distributed as dist
from ai_crypto_trader_b200.dist import gather_path_rows, shard_bounds
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
for n in (1, 2, 7, 64):                     # 1 and 2 paths: some ranks hold none
    full = torch.arange(5 * n, dtype=torch.float32).view(5, n) * 0.25 - 3.0
    lo, hi, _ = shard_bounds(n, world, rank)
    got = gather_path_rows(full[:, lo:hi].clone(), n)
    assert tuple(got.shape) == (5, n) and torch.equal(got, full), (n, rank)
if rank == 0:
    print("ROWS_OK")
dist.destroy_process_group()
'''


def test_gather_path_rows_world3_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, B200BT_ROOT=str(ROOT), MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=3",
           "--master-addr", "127.0.0.1", "--master-port", "29547", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "ROWS_OK" in res.stdout
