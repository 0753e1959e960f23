"""Throughput of VLN-CE pre-training (model/ce_pretrain.py) on one GPU: the mlm:sap 1:1 task mix of
bevbert_ce/pretrain/run_pt/r2r_pretrain_habitat.json at its 32 samples per GPU, the full-depth model of
r2r_model_config_dep.json with every dropout at 0.1 (the json's `dropout`, which train_r2r.py sets on every nn.Dropout),
whole steps replayed as CUDA graphs.  Synthetic CE batches (synth.ce_synth_config), device resident, two per task.
Device-timed over --steps steps after --warmup, as bench.py times its device-resident figure.  Prints one JSON line.

    python scripts/bench_ce.py --steps 22 --warmup 5
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MIX = ["mlm", "sap"]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(), None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--steps", type=int, default=22)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32, help="samples per step")
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_ce.py measures one GPU")
    if not torch.cuda.is_available():
        raise SystemExit("bench_ce.py needs a CUDA device: the hot path has no CPU implementation")
    from bevbert_b200 import synth
    from bevbert_b200.config import make_ce_config
    from bevbert_b200.graphs import GraphedTrainStep
    from bevbert_b200.model.ce_pretrain import GlocalTextPathCMTPreTraining
    from bevbert_b200.model.ops import prepare_batch
    from bevbert_b200.optim import AdamW, build_param_groups
    from bevbert_b200.parallel import direct_param_grads, enable_side_stream

    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    cfg = make_ce_config(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, feat_dropout=0.1)
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).to(dev).train()
    direct_param_grads(True)
    enable_side_stream(True)
    opt = AdamW(build_param_groups(model, 0.01), lr=5e-5, betas=(0.9, 0.98), eps=1e-6, max_grad_norm=5.0,
                runtime=model.rt)
    scfg = synth.ce_synth_config(batch_size=args.batch)
    batches = {t: [synth.batch_to(prepare_batch(synth.make_batch(scfg, seed=1234 + 13 * j, task=t)), dev)
                   for j in range(2)] for t in MIX}
    step = GraphedTrainStep(model, opt)
    for t in MIX:                       # two eager steps, the capture and a first replay per (task, batch)
        for j in range(2):
            for _ in range(4):
                step(batches[t][j], t)
    for i in range(args.warmup):
        step(batches[MIX[i % 2]][(i // 2) % 2], MIX[i % 2])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    loss = None
    for i in range(args.steps):
        loss = step(batches[MIX[i % 2]][(i // 2) % 2], MIX[i % 2])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    graphed = all(step.launches(batches[t][j], t) for t in MIX for j in range(2))
    name, power = gpu_info()
    print(json.dumps({"workload": "vln-ce pretrain mlm:sap 1:1", "samples_per_step": args.batch,
                      "ms_per_step": round(ms, 3), "samples_per_s": round(args.batch / ms * 1e3, 2),
                      "steps": args.steps, "warmup": args.warmup, "graphs": bool(graphed),
                      "last_loss": float(loss), "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
