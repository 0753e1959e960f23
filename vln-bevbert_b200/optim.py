"""AdamW + global-norm gradient clipping as ONE multi-tensor update over all parameters (csrc/optim.cu), with the
reference's semantics:

  * `pretrain_src/optim/adamw.py:53-112` -- per-parameter step counter (a parameter without a gradient is skipped
    entirely: no moment update, no decay, no step), m / v updates, `denom = sqrt(v) + eps` (eps OUTSIDE the sqrt,
    default 1e-6), bias-corrected step size `lr * sqrt(1 - b2^t) / (1 - b1^t)` when `correct_bias`, and the decoupled
    weight decay applied AFTER the Adam update on the updated value (`p -= lr * wd * p`);
  * `pretrain_src/optim/misc.py:12-37` -- two parameter groups, no decay for bias / LayerNorm parameters
    (`build_param_groups`);
  * `pretrain_src/train_r2r.py:295-300` -- `clip_grad_norm_(model.parameters(), grad_norm)`: every gradient is scaled by
    `min(1, max_norm / (||g||_2 + 1e-6))`; the norm is reduced and consumed on the device (no host sync) and returned
    as a 0-d tensor for logging.

The same kernel writes the bf16 shadow of every updated weight (blocks.WeightCache), so no separate re-cast pass runs
after the step.  This module only builds the launch tables; there is no PyTorch arithmetic on the parameters here.
"""
import math

import torch

from . import kernels as K

NO_DECAY = ("bias", "LayerNorm.bias", "LayerNorm.weight")


def build_param_groups(model, weight_decay):
    """pretrain_src/optim/misc.py:12-23."""
    named = list(model.named_parameters())
    return [{"params": [p for n, p in named if not any(nd in n for nd in NO_DECAY)], "weight_decay": weight_decay},
            {"params": [p for n, p in named if any(nd in n for nd in NO_DECAY)], "weight_decay": 0.0}]


class AdamW:
    """`AdamW(params_or_groups, lr, betas, eps, weight_decay, correct_bias, max_grad_norm=None, runtime=None)`.
    `runtime` (model.rt) lets the update kernel maintain the bf16 weight shadows; `param_groups` entries may carry
    their own `lr` / `weight_decay` like torch optimizers (schedulers write `group["lr"]`)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True,
                 max_grad_norm=None, runtime=None):
        params = list(params)
        if params and not isinstance(params[0], dict):
            params = [{"params": params}]
        self.param_groups = []
        self.defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, correct_bias=correct_bias)
        seen = set()
        for g in params:
            g = dict(g)
            ps = []
            for p in g["params"]:
                if p.requires_grad and id(p) not in seen:
                    seen.add(id(p))
                    ps.append(p)
            g["params"] = ps
            for k, v in self.defaults.items():
                g.setdefault(k, v)
            self.param_groups.append(g)
        self.max_grad_norm = max_grad_norm
        self.rt = runtime
        if runtime is not None:
            runtime.wc.managed = True
        self.flat = [(gi, p) for gi, g in enumerate(self.param_groups) for p in g["params"]]
        self.steps = [0] * len(self.flat)
        self.m = self.v = None
        self._sumsq = None
        self._tables = {}       # gradient signature -> (MtTable, [flat index], shadow entries fully covered)
        self.grad_norm = None   # device sum of squares of the last clipped step's gradients (total_grad_norm: its sqrt)
        self.last_sig = None

    # ------------------------------------------------------------------ state
    def _init_state(self):
        dev = self.flat[0][1].device
        sizes = [(p.numel() + 3) // 4 * 4 for _, p in self.flat]
        total = sum(sizes)
        self._mbuf = torch.zeros(total, dtype=torch.float32, device=dev)
        self._vbuf = torch.zeros(total, dtype=torch.float32, device=dev)
        self.m, self.v, off = [], [], 0
        for (_, p), n in zip(self.flat, sizes):
            self.m.append(self._mbuf[off:off + p.numel()])
            self.v.append(self._vbuf[off:off + p.numel()])
            off += n
        self._sumsq = torch.zeros(1, dtype=torch.float32, device=dev)

    def state_dict(self):
        return {"steps": list(self.steps), "exp_avg": [m.clone() for m in (self.m or [])],
                "exp_avg_sq": [v.clone() for v in (self.v or [])]}

    def load_state_dict(self, sd):
        if self.m is None:
            self._init_state()
        self.steps = list(sd["steps"])
        for dst, src in zip(self.m, sd["exp_avg"]):
            dst.copy_(src.reshape(-1))
        for dst, src in zip(self.v, sd["exp_avg_sq"]):
            dst.copy_(src.reshape(-1))

    # ------------------------------------------------------------------ step
    def _table(self, sig):
        ent = self._tables.get(sig)
        wc = self.rt.wc if self.rt is not None else None
        if ent is not None and (wc is None or ent[3] == len(wc._c)):
            return ent
        slots = wc.shadow_slots() if wc is not None else {}
        rows, written = [], set()
        for i in sig:
            p = self.flat[i][1]
            sl = slots.get(p.data_ptr(), [])
            p16 = sl[0][0] if sl else 0     # the update kernel writes ONE bf16 copy per parameter
            rows.append((p.data_ptr(), 0, self.m[i].data_ptr(), self.v[i].data_ptr(), p16, p.numel(), 0.0, 0.0))
            if sl:
                written.add((p.data_ptr(), id(sl[0][1])))
        # shadows that hold an updated parameter the kernel does not write (zero-padded tiny operands, a second shadow
        # of the same parameter): marked stale after the step, WeightCache.get re-casts them
        stale = []
        if wc is not None:
            ptrs = {self.flat[i][1].data_ptr() for i in sig}
            for e in wc.entries_with(ptrs):
                if any(q.data_ptr() in ptrs and (q.data_ptr(), id(e)) not in written for q in e.params):
                    stale.append(e)
        tab = K.MtTable(rows, self.flat[0][1].device)
        ent = (tab, list(sig), stale, len(wc._c) if wc is not None else 0)
        self._tables[sig] = ent
        return ent

    def _fill(self, tab, idx, sig, with_grads):
        """host half of a step: advance the per-parameter step counters and write step size / decay (and, outside
        graph replay, the gradient pointers) into the pinned launch table.  -> False when the table is out of date."""
        tab.wait_idle()         # an upload of the previous step of this table may still be queued: do not race it
        rows = tab.np
        for r, i in enumerate(idx):
            gi, p = self.flat[i]
            grp = self.param_groups[gi]
            if with_grads:
                g = p.grad
                if g.dtype != torch.float32 or not g.is_contiguous():
                    g = p.grad = g.float().contiguous()
                if rows["p"][r] != p.data_ptr():      # storage moved (module.to(), bias re-homing): rebuild the table
                    for j in idx[:r]:
                        self.steps[j] -= 1
                    self._tables.pop(sig, None)
                    return False
                rows["g"][r] = g.data_ptr()
            self.steps[i] += 1
            t = self.steps[i]
            lr = grp["lr"]
            b1, b2 = grp["betas"]
            rows["step_size"][r] = lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t) if grp["correct_bias"] else lr
            rows["decay"][r] = lr * grp["weight_decay"]
        return True

    @torch.no_grad()
    def step(self, grad_scale=1.0, set_to_none=True):
        from . import blocks
        blocks.join_side()      # side-stream mode: weight gradients must have landed (no-op otherwise)
        sig = tuple(i for i, (_, p) in enumerate(self.flat) if p.grad is not None)
        if not sig:
            return None
        if self.m is None:
            self._init_state()
        tab, idx, stale, _ = self._table(sig)
        if not self._fill(tab, idx, sig, True):
            return self.step(grad_scale, set_to_none)
        tab.upload()
        tab.mark_busy()
        b1, b2 = self.param_groups[0]["betas"]
        eps = self.param_groups[0]["eps"]
        clip = self.max_grad_norm is not None and self.max_grad_norm > 0
        if clip:
            K.mt_sumsq(tab, self._sumsq)
            self.grad_norm = self._sumsq
        K.adamw_step(tab, b1, b2, eps, self._sumsq if clip else None, float(self.max_grad_norm or 0.0), grad_scale)
        for e in stale:
            e.epoch = -1
        if set_to_none:
            for i in idx:
                self.flat[i][1].grad = None
        self.last_sig = sig
        return self.total_grad_norm() if clip else None

    def advance(self, sig):
        """CUDA-graph replay of a captured step(): the graph re-uploads the pinned table and re-launches the kernels;
        only the host half (step counters, bias-corrected step sizes, current lr) has to be redone before the replay."""
        tab, idx, _, _ = self._tables[sig]
        self._fill(tab, idx, sig, False)

    def replayed(self, sig):
        """call right after enqueuing a replay of a graph that holds step() of `sig`: its upload node reads the pinned
        table until the replay has passed it (MtTable.mark_busy / wait_idle)."""
        self._tables[sig][0].mark_busy()

    def total_grad_norm(self):
        """sqrt of the device-side sum of squares of the last clipped step (0-d tensor, no sync)."""
        return None if self.grad_norm is None else self.grad_norm.sqrt().reshape(())

    def zero_grad(self, set_to_none=True):
        for _, p in self.flat:
            if p.grad is not None:
                if set_to_none:
                    p.grad = None
                else:
                    p.grad.zero_()


FusedAdamW = AdamW   # round-1 name
