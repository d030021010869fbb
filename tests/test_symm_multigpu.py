"""T3 (multi-GPU): the fused RS+AdamW+AG round kernel over symmetric memory vs the NCCL path."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def test_fused_round_kernel_matches_nccl_path(tmp_path):
    n = min(torch.cuda.device_count(), 8)
    out = tmp_path / "symm.json"
    from acco_b200.launch import free_port
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "tools", "symm_check.py"), "--numel", "5000011",
           "--bench-numel", "8000000", "--bench-iters", "3", "--out", str(out)]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:]
    rep = json.load(open(out))
    assert any(v.get("available") and v.get("ok") for v in rep["modes"].values()), rep


def test_fused_allgather_gemm_training_path():
    """train.fused_ag_gemm=True (KERNEL B pulls remote weight tiles inside the first forward GEMM) == baseline training."""
    n = 2
    from acco_b200.launch import free_port
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "tools", "fused_ag_check.py")]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:]


def test_gather_gemm_kernel():
    n = min(torch.cuda.device_count(), 8)
    from acco_b200.launch import free_port
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "tools", "gather_gemm_check.py"), "--N", "4608"]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:]


def test_backends_train_to_the_same_parameters_and_tolerate_a_slow_rank(tmp_path):
    """20 ACCO rounds on symm-multimem vs symm-p2p vs nccl: ranks bit-identical, backends within bf16 tolerance; with a slowed rank
    the fast ranks accumulate more micro-batches per round and the result is still consistent (tools/train_equiv_check.py)."""
    n = min(torch.cuda.device_count(), 8)
    out = tmp_path / "equiv.json"
    from acco_b200.launch import free_port
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "tools", "train_equiv_check.py"), "--rounds", "20", "--out", str(out)]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:]
    rep = json.load(open(out))
    assert rep["ok"] and rep["checks"]["hetero"]["fast_ranks_accumulated_more"], rep
