"""bench.py in the library's deterministic mode: the same workload, arguments and JSON line, with
torch.use_deterministic_algorithms(True) set before the run and "deterministic": true added to the result.

    python scripts/bench_deterministic.py --gpus 1 --steps 22 --warmup 5 [--dump-outputs DIR]

cuBLAS (the einsum of the SAP fusion) is deterministic only with CUBLAS_WORKSPACE_CONFIG set before CUDA initialises,
so it is set here first.  torch's fill of uninitialised memory with NaNs, which the flag turns on, is turned off, so
that the measured cost is the library's.  Two runs with --dump-outputs write byte-identical files on the same build
and GPU model."""
import contextlib
import io
import json
import os
import sys

os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402


def main():
    if "reference" in sys.argv[1:]:
        raise SystemExit("the deterministic mode applies to the GPU path, not to --impl reference")
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    sys.argv = [os.path.join(ROOT, "bench.py")] + sys.argv[1:]
    out = io.StringIO()
    try:
        with contextlib.redirect_stdout(out):
            bench.main()
    finally:
        for line in out.getvalue().splitlines():
            try:
                rec = json.loads(line)
            except ValueError:
                rec = None
            if isinstance(rec, dict) and "metric" in rec:
                rec["deterministic"] = True
                line = json.dumps(rec)
            print(line)


if __name__ == "__main__":
    main()
