#!/usr/bin/env python
"""Regenerate ``tests/golden/reference_acco_trace.npy``: the parameters of the original ACCO project's own step functions
(`trainer_decoupled.communication_step` / `update_buffers_step`, CPU, gloo, world size 1) after each of 6 rounds on the toy
quadratic of ``tests/test_trainer_cpu.py::test_golden_trace_against_reference_step_functions``.

    python tools/golden_reference_trace.py --reference <checkout of the original project>
"""
import argparse
import importlib.util
import os
import socket
import sys
import types

import numpy as np
import torch
import torch.distributed as dist

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_acco_trace.npy")


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reference", required=True)
    a = p.parse_args()
    if "omegaconf" not in sys.modules:                  # imported by the original trainer, not needed by its step functions
        m = types.ModuleType("omegaconf")
        m.OmegaConf = type("OmegaConf", (), {"to_container": staticmethod(lambda c, resolve=True: dict(c))})
        sys.modules["omegaconf"] = m
    sys.path.insert(0, a.reference)
    spec = importlib.util.spec_from_file_location("_reference_trainer_decoupled", os.path.join(a.reference, "trainer_decoupled.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=0, world_size=1)
    params = torch.tensor([1.0, 2.0, 3.0, 4.0])
    k = [0]

    def grad_at(p):
        g = 0.1 * (k[0] + 1) * p
        k[0] += 1
        return g

    params.grad = grad_at(params).clone()                       # prepare_grads: g0 at theta0 (kept, not zeroed)
    com_buffer = params.grad.clone()                             # prepare_buffer_com, no warm-up: grads, count 1
    count_this_round = torch.ones(1, dtype=torch.int)
    count_local = torch.ones(1, dtype=torch.int)
    params_opt = params.clone().float()
    params_opt.grad = torch.zeros_like(params_opt)
    opt = torch.optim.AdamW([params_opt], lr=0.1, weight_decay=0.0, betas=(0.9, 0.95))
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: 1.0)
    trace = []
    for r in range(6):
        ref.communication_step(0, 4, 4, None, count_this_round, com_buffer, params_opt, opt, sched, r)
        params.grad.add_(grad_at(params))                        # main thread: one micro-batch during the round
        count_local.add_(1)
        ref.update_buffers_step(params, com_buffer, 4, count_this_round, count_local, r)
        trace.append(params.clone())
    dist.destroy_process_group()
    np.save(OUT, torch.stack(trace).numpy().astype(np.float32))
    print(OUT, torch.stack(trace))


if __name__ == "__main__":
    main()
