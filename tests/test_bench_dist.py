"""Host-side logic of bench.py's multi-process path on CPU (gloo, world size 2): barrier + MAX
reduction of the per-rank elapsed time, rank-0-only reporting, and the reference arm's rank rule."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import os, sys, json
sys.path.insert(0, %r)
import torch, torch.distributed as dist
import bench
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
t = bench.max_over_ranks(0.5 + rank, torch.device("cpu"), world)       # ranks report 0.5 s and 1.5 s
agg = bench.aggregate_value(10, t, world)
dist.barrier()
if rank == 0:
    print(json.dumps({"t": t, "value": agg}))
dist.destroy_process_group()
''' % ROOT


def test_max_over_ranks_and_aggregate(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29613", str(script)], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    line = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(line) == 1, r.stdout          # only rank 0 prints
    out = json.loads(line[0])
    assert abs(out["t"] - 1.5) < 1e-9        # MAX over ranks
    assert abs(out["value"] - 2 * 10 / 1.5) < 1e-9   # whole-job frames/s: world * steps / max time


def test_reference_arm_other_ranks_exit_silently():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=120, env=env, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_reference_arm_rank0_prints_the_contract_line():
    """`bench.py --impl reference` on rank 0: one JSON line with the arm's keys, measured on the CPU oracle (runs here)."""
    env = dict(os.environ, RANK="0", WORLD_SIZE="1", LOCAL_RANK="0")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0", "--ref-threads", "2"],
                       capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    out = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "config", "cpu_baseline", "e2e"):
        assert k in out, k
    assert out["impl"] == "reference" and out["unit"] == "frames/s" and out["value"] > 0
    assert out["cpu_baseline"]["kind"] == "port" and out["cpu_baseline"]["cores"] == 2 and out["cpu_baseline"]["value"] == out["value"]
    assert out["e2e"] == {"value": out["value"], "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


DUMP_WORKER = r'''
import os, sys
sys.path.insert(0, %r)
import numpy as np, torch.distributed as dist
import bench
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")


class Stream:                      # stands in for bench.CameraStream: 100 bytes of rank- and stream-specific outputs
    def __init__(self, sid):
        self.sid = sid

    def last_outputs(self):
        return {"keypoints": np.full(25, 10 * rank + self.sid, np.float32)}


bench.DUMP_LIMIT_BYTES = 500       # 250 bytes per rank: two of the three streams fit
dist.barrier()
bench.dump_outputs(sys.argv[1], [Stream(s) for s in range(3)], rank, world)
dist.barrier()
dist.destroy_process_group()
''' % ROOT


def test_dump_outputs_two_ranks(tmp_path):
    """--dump-outputs under two processes: each rank writes its own files, and the cap holds for the whole job."""
    script = tmp_path / "worker.py"
    script.write_text(DUMP_WORKER)
    out = tmp_path / "dump"
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29614", str(script), str(out)], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    files = sorted(os.listdir(out))
    assert files == ["r%d_s%d_keypoints.npy" % (k, s) for k in (0, 1) for s in (0, 1)]
    import numpy as np
    for f in files:
        k, s = int(f[1]), int(f[4])
        assert np.array_equal(np.load(out / f), np.full(25, 10 * k + s, np.float32))
    assert sum(os.path.getsize(out / f) for f in files) <= 500 + 4 * 128     # 4 x 100 data bytes + .npy headers
