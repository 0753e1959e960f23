"""Per-kernel cost of the deterministic mode: torch.profiler CUDA time of the R2R pre-training step (bench.py's
headline workload, eager launches, side stream on) with torch.use_deterministic_algorithms off and on, summed per
kernel name over one task cycle; prints the kernels whose time changed most."""
import os
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402
from bevbert_b200 import blocks as Bk, synth  # noqa: E402
from bevbert_b200.model.ops import prepare_batch  # noqa: E402
from bevbert_b200.model.pretrain_cmt import GlocalTextPathCMTPreTraining  # noqa: E402
from bevbert_b200.optim import AdamW, build_param_groups  # noqa: E402
from bevbert_b200.parallel import direct_param_grads, enable_side_stream  # noqa: E402


def main():
    torch.manual_seed(0)
    model = synth.det_init_(GlocalTextPathCMTPreTraining(bench.full_config()), seed=3).cuda().train()
    direct_param_grads(True)
    enable_side_stream(True)
    opt = AdamW(build_param_groups(model, 0.01), lr=5e-5, betas=(0.9, 0.98), eps=1e-6, max_grad_norm=5.0, runtime=model.rt)
    mix = bench.MIX
    batches = {t: synth.batch_to(prepare_batch(synth.make_batch(bench.synth_config(32), seed=1234, task=t)), "cuda")
               for t in set(mix)}

    def cycle():
        for t in mix:
            model(batches[t], t).mean().backward()
            Bk.join_side()
            opt.step()
            opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize()

    per = {}
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        torch.utils.deterministic.fill_uninitialized_memory = False
        cycle()
        cycle()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            cycle()
        per[det] = {e.key: e.device_time_total for e in prof.key_averages()}
    tot = {d: sum(v.values()) / 1e3 for d, v in per.items()}
    print("%s: CUDA kernel time per %d-step cycle: default %.1f ms, deterministic %.1f ms (%+.1f %%)" % (
        torch.cuda.get_device_name(), len(mix), tot[False], tot[True], 100.0 * (tot[True] / tot[False] - 1.0)))
    names = set(per[False]) | set(per[True])
    rows = sorted(names, key=lambda n: -abs(per[True].get(n, 0.0) - per[False].get(n, 0.0)))
    for n in rows[:20]:
        a, b = per[False].get(n, 0.0) / 1e3, per[True].get(n, 0.0) / 1e3
        print("%+9.2f ms  %8.2f -> %8.2f  %s" % (b - a, a, b, n[:110]))


if __name__ == "__main__":
    main()
