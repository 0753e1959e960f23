"""Per-step time of the VLN-CE global-map image glue, reference torch glue vs graphs.install_ce_gmap_features, over
15-step episodes (tests/ce_gmap_cases.py) at B = 1, 4 and 8, in training (with the backward of the teacher-forced loss)
and in eval (no_grad).  Both arms run the same stand-in panorama / navigation calls, so the difference between them is
the glue: the masked mean, the candidate rows, update_graph's merges, get_node_embeds, stack, pad and their backward.
The arms alternate over windows; the table gives the min-max over windows of ms per step.  Prints the card's name and
power limit from the same run, and one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ce_gmap_cases as C  # noqa: E402
from bevbert_b200 import graphs  # noqa: E402


def episode(trainer, B, train, seed):
    sched = [B] * 15
    if train:
        trainer.policy.net.zero_grad(set_to_none=True)
        _, _, loss = C.rollout(trainer, seed, schedule=sched, train=True)
        loss.backward()
    else:
        with torch.no_grad():
            C.rollout(trainer, seed, schedule=sched, train=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=6)
    ap.add_argument("--episodes", type=int, default=4)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ce_gmap.py needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    ref = C.Trainer(3, "cuda")
    ins = C.Trainer(3, "cuda")
    graphs.install_ce_gmap_features(ins)
    rows = []
    for train in (True, False):
        for B in (1, 4, 8):
            times = {"reference": [], "installed": []}
            for name, t in (("reference", ref), ("installed", ins)):
                episode(t, B, train, 0)                         # warm-up
            for w in range(a.windows):
                for name, t in (("reference", ref), ("installed", ins)) if w % 2 == 0 else \
                        (("installed", ins), ("reference", ref)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for e in range(a.episodes):
                        episode(t, B, train, 100 + e)
                    torch.cuda.synchronize()
                    times[name].append((time.perf_counter() - t0) * 1e3 / (a.episodes * 15))
            row = {"mode": "train" if train else "eval", "B": B}
            for k, v in times.items():
                row[k] = [round(min(v), 3), round(max(v), 3)]
            rows.append(row)
            print("%-5s B=%d  reference %.3f-%.3f ms/step  installed %.3f-%.3f ms/step" % (
                row["mode"], B, *row["reference"], *row["installed"]))
    print(json.dumps({"card": q, "ms_per_step": rows}))


if __name__ == "__main__":
    main()
