"""Per-kernel CUDA time of bench.py's flagship workload: torch.profiler over one default-mode task cycle of the R2R
pre-training step (same set-up as scripts/prof_det.py), summed per kernel name, with each kernel's share of the
cycle's kernel time and the share of the attention kernels (csrc/attn_tc.cu, csrc/attn_flash.cu, csrc/attn_scores.cu)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from prof_det import make_cycle  # noqa: E402

ATTN = ("attn_tc_", "flash_", "attn_scores")


def main(top=int(sys.argv[1]) if len(sys.argv) > 1 else 30):
    cycle = make_cycle()
    cycle()
    cycle()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cycle()
    per = {e.key: e.device_time_total / 1e3 for e in prof.key_averages() if e.device_time_total > 0}
    tot = sum(per.values())
    attn = {n: t for n, t in per.items() if any(a in n for a in ATTN)}
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        card = "power limit not available"
    print("%s (%s): CUDA kernel time per task cycle %.2f ms; attention kernels %.2f ms = %.1f %%" % (
        torch.cuda.get_device_name(), card, tot, sum(attn.values()), 100.0 * sum(attn.values()) / tot))
    for n, t in sorted(attn.items(), key=lambda kv: -kv[1]):
        print("  attn %8.3f ms %5.1f %%  %s" % (t, 100.0 * t / tot, n[:100]))
    for n, t in sorted(per.items(), key=lambda kv: -kv[1])[:top]:
        print("%8.3f ms %5.1f %%  %s" % (t, 100.0 * t / tot, n[:110]))


if __name__ == "__main__":
    main()
