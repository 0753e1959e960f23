"""Whole-step CUDA-graph replay for the pre-training loop: forward + backward (+ gradient all-reduce) + optimizer of one
(task, batch-shape) is captured once and replayed, so a step costs the host one `cudaGraphLaunch` instead of ~600 kernel
launches plus the Python block / autograd glue (eager stepping spends that much host time per step whatever the kernels
do).

What makes a step replayable here:
  * inputs live in STATIC device tensors (the caller refills them in place, e.g. from pinned host memory on a copy
    stream -- bench.py's `dev_in` buffers); host-side index lists come from `ops.prepare_batch` (pinned tensors that
    the captured copy nodes re-read);
  * dropout seeds are kernel parameters frozen in the graph, so the per-step variation comes from the device-resident
    salt every kernel XORs into its seed (`bb_set_drop_salt_ptr`); the salt is advanced ON THE DEVICE (a 64-bit LCG
    step, the first two nodes of the graph), so the mask sequence does not depend on how far the host runs ahead;
  * the optimizer's host half (per-parameter step counters, bias-corrected step sizes, lr schedule) is redone before
    each replay by `optim.AdamW.advance`; the graph re-uploads the pinned launch table and runs the update kernels.
    The host may not rewrite that table while a replay that still has to read it is queued: `AdamW.replayed` records
    an event behind each replay and the next `advance` of the same table waits for it (kernels.MtTable);
  * parameter gradients are carved from the per-step arena inside the graph's memory pool: same addresses every replay.
A graph is keyed by (task, identity and shapes of the batch tensors).  sem / masksem, whose per-item loss has a
device-computed length, run in the model's `sync_free_mean` mode (mean over a device-side weight, same value and
gradients); a step whose capture fails (a host synchronisation somewhere in forward) falls back to eager launches.
"""
import torch

from . import blocks
from . import kernels as K
from . import _lib

EAGER_TASKS = ()      # every pre-training task is capturable (sem / masksem through the model's sync_free_mean mode)


_SALT = {}      # device -> device word: registered with the library once and never freed
_LCG_A, _LCG_C = 6364136223846793005, 1442695040888963407      # Knuth's MMIX multiplier / increment (mod 2^64)


def _salt_buffers(dev):
    key = (dev.type, dev.index)
    if key not in _SALT:
        word = torch.zeros(1, dtype=torch.int64, device=dev)
        _lib.check(_lib.load().bb_set_drop_salt_ptr(word.data_ptr()), "bb_set_drop_salt_ptr")
        _SALT[key] = word
    return _SALT[key]


class GraphedTrainStep:
    def __init__(self, net, optimizer, reduce_grads=None, warmup=2, loss_fn=None):
        self.net, self.opt, self.reduce_grads, self.warmup = net, optimizer, reduce_grads, warmup
        self.loss_fn = loss_fn or (lambda out: out.mean())
        self.entries = {}
        self.pool = None
        dev = next(net.parameters()).device
        self.salt_dev = _salt_buffers(dev)
        _lib.check(_lib.load().bb_set_drop_salt_ptr(self.salt_dev.data_ptr()), "bb_set_drop_salt_ptr")
        # reproducible mask sequence: the salt restarts from the process seed for every training loop
        self.salt_dev.fill_(blocks._mix64(torch.initial_seed() + 0x5A17) & 0x7FFFFFFFFFFFFFFF)
        self.launches_per_replay = {}

    @staticmethod
    def _sig(batch, task):
        return (task, id(batch)) + tuple((k, v.data_ptr(), tuple(v.shape)) for k, v in sorted(batch.items())
                                         if torch.is_tensor(v))

    def _forward(self, batch, task):
        mod = self.net.module if hasattr(self.net, "module") else self.net
        if task.startswith(("sem", "masksem")) and hasattr(mod, "sync_free_mean"):
            mod.sync_free_mean = True
            try:
                return self.net(batch, task)
            finally:
                mod.sync_free_mean = False
        return self.net(batch, task)

    def _eager(self, batch, task, like_replay=False):
        """one step with eager launches.  `like_replay` (data-parallel, this rank's capture failed): issue the same
        collectives as the ranks that replay a graph -- ONE all-reduce of the whole arena after backward instead of the
        chunked ones the backward hook would launch -- so that the ranks stay in step."""
        rg = self.reduce_grads
        chunked = getattr(rg, "enabled", None)
        if like_replay and chunked is not None:
            rg.enabled = False
        try:
            loss = self.loss_fn(self._forward(batch, task))
            loss.backward()
        finally:
            if like_replay and chunked is not None:
                rg.enabled = chunked
        if rg is not None:
            rg()
        self.opt.step()
        return loss.detach()

    def _next_salt(self):
        """advance the device-resident dropout salt: enqueued eagerly, or recorded as the first nodes of a step graph"""
        self.salt_dev.mul_(_LCG_A).add_(_LCG_C)

    def __call__(self, batch, task):
        if EAGER_TASKS and task.startswith(EAGER_TASKS):
            self._next_salt()
            return self._eager(batch, task)
        key = self._sig(batch, task)
        ent = self.entries.get(key)
        if ent is None:
            ent = self.entries[key] = {"n": 0, "graph": None}
        if ent["graph"] is None and ent["n"] < self.warmup:
            ent["n"] += 1
            self._next_salt()
            return self._eager(batch, task)
        if ent["graph"] is None and ent.get("failed"):
            self._next_salt()
            return self._eager(batch, task, like_replay=True)
        if ent["graph"] is not None and self.reduce_grads is not None:
            # data-parallel: the graph holds forward + backward; the NCCL all-reduce and the optimizer run eagerly on the
            # gradients the graph left in its (static) arena.  Collectives stay out of the capture: a rank whose capture
            # failed would execute them while the others only record them, and capturing the chunked reductions on the
            # communication stream faulted in an earlier two-GPU experiment (illegal address at the first replay).
            ent["graph"].replay()
            self._after_backward_eager(ent)
            return ent["loss"]
        if ent["graph"] is None:
            try:
                self._capture(ent, batch, task)
            except Exception as e:          # e.g. a host sync inside forward: this (task, batch) stays eager
                import warnings
                warnings.warn("CUDA-graph capture of the %s step failed (%s: %s); running it eagerly" % (
                    task, type(e).__name__, str(e)[:200]))
                torch.cuda.synchronize()
                ent["failed"] = True
                for p in self.net.parameters():
                    p.grad = None
                self._next_salt()
                return self._eager(batch, task, like_replay=True)
        else:
            self.opt.advance(ent["sig"])
            ent["graph"].replay()
            self.opt.replayed(ent["sig"])
        return ent["loss"]

    def _after_backward_eager(self, ent):
        """data-parallel replay: hand the graph's gradient tensors back to the parameters, then all-reduce + step"""
        A = blocks.ARENA
        A.buf, A.off, A.need, A.tag = ent["arena"]
        A.step_id += 1
        for p, g in ent["grads"]:
            p.grad = g
        blocks.PENDING_ADDS[:] = ent["pending"]
        self.reduce_grads()
        self.opt.step()

    def _capture(self, ent, batch, task):
        for p in self.net.parameters():
            p.grad = None
        torch.cuda.synchronize()
        if self.pool is None:
            self.pool = torch.cuda.graph_pool_handle()
        g = torch.cuda.CUDAGraph()
        n0 = K.launch_count()
        dp = self.reduce_grads is not None
        hook, blocks.AFTER_BLOCK_BWD = blocks.AFTER_BLOCK_BWD, (None if dp else blocks.AFTER_BLOCK_BWD)
        try:
            with torch.cuda.graph(g, pool=self.pool):
                self._next_salt()
                loss = self.loss_fn(self._forward(batch, task))
                loss.backward()
                if dp:
                    blocks.join_side()       # side-stream work rejoins inside the graph; gradients stay in the arena
                else:
                    self.opt.step()
                ent["loss"] = loss.detach()
        finally:
            blocks.AFTER_BLOCK_BWD = hook
        ent["launches"] = K.launch_count() - n0
        ent["graph"] = g
        if dp:
            params = [p for p in self.net.parameters() if p.grad is not None]
            ent["grads"] = [(p, p.grad) for p in params]
            ent["pending"] = list(blocks.PENDING_ADDS)
            A = blocks.ARENA
            ent["arena"] = (A.buf, A.off, A.need, A.tag)
            g.replay()                       # the capture only RECORDED forward + backward: run them once
            self._after_backward_eager(ent)
        else:
            ent["sig"] = self.opt.last_sig
            # the capture only RECORDED the step (and advanced the optimizer's host counters for it): run it once
            g.replay()
            self.opt.replayed(ent["sig"])

    def launches(self, batch, task):
        """kernels of libbevbert_b200.so inside the captured step of (batch, task), or None when it runs eagerly."""
        ent = self.entries.get(self._sig(batch, task))
        return ent.get("launches") if ent and ent.get("graph") is not None else None
