"""The VLN-CE model under the flat gradient all-reduce of bevbert_b200/parallel.py (gloo, world size 2, kernels
emulated): two ranks on half batches give the gradients of one process on the whole batch, on the step arena."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))


def _worker(rank, world, port, task, ret):
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, HERE)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), BEVBERT_CHECK_ARENA="1")
    torch.set_num_threads(2)
    import ce_cases
    import emu_kernels
    emu_kernels.install()
    import bevbert_b200.kernels as K
    K.add_rows = ce_cases.emu_add_rows(emu_kernels.add_rows)
    from bevbert_b200 import blocks, synth
    from bevbert_b200.config import make_ce_config
    from bevbert_b200.model.ce_pretrain import GlocalTextPathCMTPreTraining
    from bevbert_b200.parallel import FlatGradAllReduce, broadcast_parameters
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cfg = make_ce_config(small=True)
    full = synth.make_batch(synth.ce_synth_config(batch_size=4, pano_min=3, pano_max=5, gmap_min=6, gmap_max=8), seed=9,
                            task=task)
    shard = synth.split_batch(full, world)[rank]
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).train()
    broadcast_parameters(model)
    reducer = FlatGradAllReduce(model.parameters(), world)
    for _ in range(2):          # the second step runs on the step arena (reduced in place)
        model.zero_grad(set_to_none=True)
        model(synth.clone_batch(shard), task).mean().backward()
        reducer()
    assert blocks.ARENA.buf is not None and blocks.ARENA.off > 0
    grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    if rank == 0:
        single = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).train()
        single(full, task).mean().backward()
        ref = {n: p.grad for n, p in single.named_parameters() if p.grad is not None}
        top = max(float(g.norm()) for g in ref.values())
        assert set(ref) == set(grads), set(ref) ^ set(grads)
        ret["worst"] = max(float((grads[n] - g).norm()) / max(float(g.norm()), 1e-4 * top) for n, g in ref.items())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("task", ["mlm", "sap"])
def test_flat_all_reduce_gradients_equal_single_process(task):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, port, task, ret), nprocs=2, join=True)
    assert ret["worst"] < 1e-3, ret["worst"]
