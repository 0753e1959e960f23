"""The VLN-CE trainer's global-map image input, `gmap_img_fts`, from a device-resident node-embedding memory.

The reference builds it in four places every step (bevbert_ce/vlnce_baselines/ss_trainer_BEV.py and
models/graph_utils.py): the rollout's masked mean of the `panorama` call's `pano_embeds` (lines 1032-1033), the
candidate rows `pano_embeds[i][nav_types[i] == 1]` (lines 1060-1066, one host synchronisation per environment),
`GraphMap.update_graph`'s ghost sums (one launch per merge) and `_nav_gmap_variable`'s division, `torch.stack` and
`pad_tensors_wgrad` (lines 534-611), all replayed op by op by the backward.  Here the episode's `panorama` outputs stay
where the network wrote them (`Memory`, one per episode), the `GraphMap`s hold small handles to their rows instead of
tensors (`Node`, `Cands`), and each `navigation` call builds the padded (B, G, 768) fp32 input with one
`bb_ce_gmap_features` launch over an int32 table staged by one host-to-device copy; its backward is one
`bb_ce_gmap_features_bwd` launch that writes the gradient of every stored step's `pano_embeds`.

`graphs.install_ce_gmap_features(trainer)` installs it on a trainer; the arithmetic is documented at the entry points
in include/bevbert_b200.h.
"""
import numpy as np
import torch

from . import _lib
from .kernels import _stream

MAX_VIEWS = 63      # bb_ce_gmap_features reproduces torch's CUDA sum over the views below 64 views
_PLACEHOLDER = torch.zeros(0)


class Node:
    """GraphMap.node_embeds entry: the masked mean of row i of step s's pano_embeds"""
    __slots__ = ("mem", "s", "i")

    def __init__(self, mem, s, i):
        self.mem, self.s, self.i = mem, s, i


class Cands:
    """GraphMap.ghost_embeds[g][0] entry: the sum of candidate rows (s, i, k), k-th nav_types == 1 view of row i of step
    s, in merge order.  `+` is update_graph's merge; `/ count` is get_node_embeds' mean, kept lazy."""
    __slots__ = ("mem", "terms")

    def __init__(self, mem, terms):
        self.mem, self.terms = mem, terms

    def __add__(self, other):
        return Cands(self.mem, self.terms + other.terms)

    def __truediv__(self, count):
        if count != len(self.terms):
            raise ValueError("ghost count %d does not match its %d merged candidates" % (count, len(self.terms)))
        return self


class Memory:
    """One episode's `panorama` outputs (pano_embeds (B_s, V_s, H) fp32, nav_types (B_s, V_s) int64, pano_masks
    (B_s, V_s) bool, s = step - 1), referenced, not copied."""

    def __init__(self):
        self.steps = []
        self.collect = None     # while the trainer's own _nav_gmap_variable runs: GraphMap id -> its handles

    def record(self, pano, nav_types, masks):
        if not (pano.is_cuda and pano.dtype == torch.float32 and pano.dim() == 3 and pano.is_contiguous()):
            raise TypeError("pano_embeds must be a contiguous (B, V, H) fp32 CUDA tensor")
        if pano.data_ptr() % 16:
            raise ValueError("pano_embeds must start 16-byte aligned (the kernels read and write its rows as float4)")
        B, V, H = pano.shape
        if V > MAX_VIEWS or H % 4 or (self.steps and H != self.steps[0][0].shape[2]):
            raise ValueError("pano_embeds (%d, %d, %d): at most %d views, H a multiple of 4 and fixed per episode"
                             % (B, V, H, MAX_VIEWS))
        for t, dt, name in ((nav_types, torch.int64, "nav_types"), (masks, torch.bool, "pano_masks")):
            if t.dtype != dt or tuple(t.shape) != (B, V) or t.device != pano.device or not t.is_contiguous():
                raise TypeError("%s must be a contiguous (%d, %d) %s tensor on %s" % (name, B, V, dt, pano.device))
        self.steps.append((pano, nav_types, masks))

    def _step_words(self, bufs):
        """S step records (bb_ce_gmap_features): pointer pairs lo / hi, then B_s, V_s"""
        w = np.zeros((len(self.steps), 4), np.int64)
        for s, ((p, n, m), b) in enumerate(zip(self.steps, bufs)):
            w[s] = (0 if b is None else b.data_ptr(), n.data_ptr(), m.data_ptr(), p.shape[0] | (p.shape[1] << 32))
        return w.view(np.int32).reshape(-1)

    def features(self, rows):
        """rows[b]: the handles of environment b's nodes then ghosts (row 0 excluded) -> (B, G, H) fp32, zeros in row 0
        and past each environment's rows; differentiable with respect to every stored pano_embeds"""
        return _Features.apply(self, rows, *[p for p, _, _ in self.steps])


def _upload(words, device):
    return torch.from_numpy(np.ascontiguousarray(words, np.int32)).pin_memory().to(device, non_blocking=True)


class _Features(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mem, rows, *panos):
        B, G, H = len(rows), 1 + max(len(r) for r in rows), panos[0].shape[2]
        table = np.zeros((B, G, 3), np.int32)
        terms = []
        for b, hs in enumerate(rows):
            for r, h in enumerate(hs, 1):
                if h.mem is not mem:
                    raise ValueError("a handle of another episode's memory")
                if isinstance(h, Node):
                    table[b, r] = (1, h.s, h.i)
                else:
                    table[b, r] = (2, len(terms), len(h.terms))
                    terms.extend(h.terms)
        words = np.concatenate([mem._step_words(panos), table.reshape(-1), np.asarray(terms, np.int32).reshape(-1)])
        out = torch.empty(B, G, H, dtype=torch.float32, device=panos[0].device)
        dev_table = _upload(words, out.device)
        _lib.check(_lib.load().bb_ce_gmap_features(dev_table.data_ptr(), len(panos), B, G, H, out.data_ptr(),
                                                   _stream()), "bb_ce_gmap_features")
        ctx.mem, ctx.rows = mem, rows
        return out

    @staticmethod
    def backward(ctx, dout):
        mem, rows = ctx.mem, ctx.rows
        dout = dout.contiguous()
        B, G, H = dout.shape
        grads = [torch.empty_like(p) if need else None for (p, _, _), need in zip(mem.steps, ctx.needs_input_grad[2:])]
        node, cand = {}, {}
        for b, hs in enumerate(rows):
            for r, h in enumerate(hs, 1):
                if isinstance(h, Node):
                    node[h.s, h.i] = (b, r)
                else:
                    for s, i, k in h.terms:
                        cand.setdefault((s, i), {})[k] = (b, r, len(h.terms))
        recs, cands = [], []
        for s, ((p, _, _), g) in enumerate(zip(mem.steps, grads)):
            if g is None:
                continue
            for i in range(p.shape[0]):
                ks = cand.get((s, i), {})
                n = max(ks) + 1 if ks else 0
                recs.append((s, i) + node.get((s, i), (-1, -1)) + (len(cands), n))
                cands.extend(ks.get(k, (-1, -1, 0)) for k in range(n))
        words = np.concatenate([mem._step_words(grads), np.asarray(recs, np.int32).reshape(-1),
                                np.asarray(cands, np.int32).reshape(-1)])
        dev_table = _upload(words, dout.device)
        vmax = max(p.shape[1] for p, _, _ in mem.steps)
        _lib.check(_lib.load().bb_ce_gmap_features_bwd(dev_table.data_ptr(), len(mem.steps), len(recs), vmax, G, H,
                                                       dout.data_ptr(), _stream()), "bb_ce_gmap_features_bwd")
        return (None, None) + tuple(grads)


def episode(gmaps):
    """The Memory shared by the GraphMaps `gmaps` (one episode's), or None when none of them has one yet"""
    mems = {id(getattr(g, "_ce_gmap_memory", None)): getattr(g, "_ce_gmap_memory", None) for g in gmaps}
    if len(mems) != 1:
        raise RuntimeError("the trainer's GraphMaps do not belong to one episode of the installed memory")
    return next(iter(mems.values()))


def attach(trainer, gmap, mem):
    """Routes one GraphMap's embeddings to `mem`: update_graph stores a Node and one Cands per candidate instead of the
    rollout's tensors (step s = step_id - 1, row i = the GraphMap's place in trainer.gmaps), then runs the original;
    get_node_embeds returns the row bb_ce_gmap_features computes, or, while `trainer_method` runs the trainer's own
    _nav_gmap_variable, collects the handle and returns a CPU placeholder."""
    update, get = gmap.update_graph, gmap.get_node_embeds

    def update_graph(prev_vp, step_id, cur_vp, cur_pos, cur_embeds, cand_vp, cand_pos, cand_embeds, cand_real_pos):
        s = step_id - 1
        if s != len(mem.steps) - 1:
            raise RuntimeError("update_graph at step %d, but the memory holds %d panorama calls"
                               % (step_id, len(mem.steps)))
        i = next(j for j, g in enumerate(trainer.gmaps) if g is gmap)
        return update(prev_vp, step_id, cur_vp, cur_pos, Node(mem, s, i), cand_vp, cand_pos,
                      [Cands(mem, ((s, i, k),)) for k in range(len(cand_vp))], cand_real_pos)

    def get_node_embeds(vp):
        h = get(vp)
        if mem.collect is None:
            return mem.features([[h]])[0, 1]
        mem.collect.setdefault(id(gmap), []).append(h)
        return _PLACEHOLDER

    gmap._ce_gmap_memory = mem
    gmap.update_graph, gmap.get_node_embeds = update_graph, get_node_embeds


def trainer_method(original, gmaps, *args):
    """Runs the trainer's own _nav_gmap_variable(*args) over the attached GraphMaps `gmaps` with placeholder embeddings
    -> (its dict, the handles each GraphMap's get_node_embeds gave, in the method's own order)"""
    mem = episode(gmaps)
    mem.collect = {}
    try:
        out = original(*args)
        rows = [mem.collect.get(id(g), []) for g in gmaps]
    finally:
        mem.collect = None
    return out, rows
