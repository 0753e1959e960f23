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

`GraphedNavigation` (below) replays the agents' per-step inference calls the same way, over padded shape buckets,
`install_ce_replay` the VLN-CE policy's, `install_ce_rgb_encoder` the CE policy's CLIP RGB encoder,
`install_ce_depth_encoder` its ResNet-50 depth encoder, and `install_ce_waypoint_predictor` the CE trainer's waypoint
predictor.  `install_ce_gmap_features` builds the CE trainer's global-map image input on the kernels (no replay).
`install_ce_lift` runs the CE trainer's `lift` (node point clouds) on the kernels (no replay).
"""
import functools

import torch

from . import blocks
from . import kernels as K
from . import _lib
from .model import ops

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


# =============================================================================================== agent per-step API
# Inputs of GlocalTextPathNavCMT.forward(mode, batch) and the dimensions of each that are padded to a multiple of 8 in
# a graph's static buffers.  Every padding value is zero / False: masks False, ids / features / pair distances 0,
# visited False, candidate index 0 (cell 0).  The model turns False masks into -10000 (text, map, BEV keys) or -inf
# (panorama keys) and -inf logits, so real rows see exact zeros from padded slots.
NAV_PAD_DIMS = {
    "language": {"txt_ids": (1,), "txt_masks": (1,)},
    "panorama": {"view_img_fts": (1,), "obj_img_fts": (1,), "loc_fts": (1,), "nav_types": (1,), "view_lens": (),
                 "obj_lens": ()},
    "navigation": {"txt_embeds": (1,), "txt_masks": (1,), "gmap_img_embeds": (1,), "gmap_step_ids": (1,),
                   "gmap_pos_fts": (1,), "gmap_masks": (1,), "gmap_pair_dists": (1, 2), "gmap_visited_masks": (1,),
                   "bev_fts": (), "bev_pos_fts": (), "bev_masks": (), "bev_nav_masks": (), "bev_cand_idxs": (1,),
                   "obj_embeds": (1,), "obj_masks": (1,)},
}


def _round8(n):
    return (n + 7) // 8 * 8


def _bucket(dims, mode, batch):
    key = [mode, torch.are_deterministic_algorithms_enabled()]
    for name, d in dims[mode].items():
        x = batch.get(name)
        if x is None:
            key.append(None)
        else:
            key.append((tuple(_round8(n) if i in d else n for i, n in enumerate(x.shape)), x.dtype))
    return tuple(key)


def _pad(dims, mode, batch, device):
    out = {}
    for name, k in zip(dims[mode], _bucket(dims, mode, batch)[2:]):
        if k is not None:
            out[name] = torch.zeros(k[0], dtype=k[1], device=device)
            out[name][tuple(slice(0, n) for n in batch[name].shape)] = batch[name]
    return out


def nav_bucket(mode, batch):
    """Graph key of a per-step call: mode, deterministic flag, and the padded shape and dtype of every input (B, object
    presence, instruction length, map nodes, BEV candidates, object and panorama tokens)."""
    return _bucket(NAV_PAD_DIMS, mode, batch)


def nav_pad(mode, batch, device):
    """The padded inputs a replay of `batch` computes on, as new zero-padded device tensors."""
    return _pad(NAV_PAD_DIMS, mode, batch, device)


def nav_slice(mode, out, batch):
    """Outputs of a padded call cut back to the caller's shapes, as fresh tensors."""
    c = torch.Tensor.clone
    if mode == "language":
        return c(out[:, :batch["txt_ids"].shape[1]])
    if mode == "panorama":
        T = batch["loc_fts"].shape[1]            # = the view width, or max(view + object lens) with objects
        return c(out[0][:, :T]), c(out[1][:, :T])
    G, Kc = batch["gmap_masks"].shape[1], batch["bev_cand_idxs"].shape[1]
    res = {"gmap_embeds": c(out["gmap_embeds"][:, :G]), "global_logits": c(out["global_logits"][:, :G]),
           "local_logits": c(out["local_logits"][:, :Kc]), "fused_logits": c(out["fused_logits"][:, :G]),
           "obj_logits": None}
    if out["obj_logits"] is not None:
        res["obj_logits"] = c(out["obj_logits"][:, :batch["obj_masks"].shape[1]])
    return res


def nav_forward_padded(model, mode, pad, host=None):
    """model on padded inputs `pad` (nav_pad).  Navigation takes the viewpoint-id lists of the caller's batch in `host`:
    a (gmap_vpids, bev_cand_vpids) pair, where gmap_vpids may be a PreparedList with staged fusion matches."""
    if mode == "language":
        return model.forward_text(pad["txt_ids"], pad["txt_masks"])
    if mode == "panorama":
        return model.forward_panorama_per_step(pad["view_img_fts"], pad.get("obj_img_fts"), pad["loc_fts"],
                                               pad["nav_types"], pad["view_lens"], pad.get("obj_lens"),
                                               vtot=pad["loc_fts"].shape[1])
    p = pad
    return model.forward_navigation_per_step(
        p["txt_embeds"], p["txt_masks"], p["gmap_img_embeds"], p["gmap_step_ids"], p["gmap_pos_fts"], p["gmap_masks"],
        p["gmap_pair_dists"], p["gmap_visited_masks"], host[0], p["bev_fts"], p["bev_pos_fts"], p["bev_masks"],
        p["bev_nav_masks"], p["bev_cand_idxs"], host[1], p.get("obj_embeds"), p.get("obj_masks"))


class Surface:
    """What GraphedNavigation needs to know about one per-step API: the padded dimensions of each call's inputs
    (`dims`), the model on padded inputs (`padded(model, mode, pad, host)`), the outputs cut back to the caller's
    shapes (`slice(mode, out, batch)`) and the unwrapped call (`eager(model, mode, batch)`).  `grad_ok`: eval-mode
    calls replay with grad enabled too (a frozen, forward-only model); `stale(model)`: True when the weights changed
    since the previous call, so that every call, not only `language`, re-casts the shadows first.  `shape_key(mode,
    batch)`: hashable sizes of a call that its inputs' shapes do not show; they join the bucket key and reach `padded`
    as `host`."""

    def __init__(self, dims, padded, slice, eager, grad_ok=False, stale=None, shape_key=None):
        self.dims, self.padded, self.slice, self.eager = dims, padded, slice, eager
        self.grad_ok, self.stale, self.shape_key = grad_ok, stale, shape_key


NAV = Surface(NAV_PAD_DIMS, nav_forward_padded, nav_slice,
              lambda model, mode, batch: type(model).forward(model, mode, batch))


# ------------------------------------------------------------------------------------ VLN-CE policy (model/ce_nav.py)
# The CE policy calls three methods of its network; each is one mode here, its arguments the batch's keys.
CE_NAV_CALLS = {
    "forward_txt": ("language", ("txt_ids", "txt_masks")),
    "forward_panorama": ("panorama", ("rgb_fts", "dep_fts", "loc_fts", "nav_types", "view_lens")),
    "forward_navigation": ("navigation", ("txt_embeds", "txt_masks", "gmap_vpids", "gmap_step_ids", "gmap_img_fts",
                                          "gmap_pos_fts", "gmap_masks", "gmap_visited_masks", "gmap_pair_dists",
                                          "bev_fts", "bev_pos_fts", "bev_masks", "bev_nav_masks", "bev_cand_idxs",
                                          "bev_cand_vpids")),
}
_CE_METHOD = {mode: name for name, (mode, _) in CE_NAV_CALLS.items()}
CE_NAV_PAD_DIMS = {
    "language": {"txt_ids": (1,), "txt_masks": (1,)},
    "panorama": {"rgb_fts": (1,), "dep_fts": (1,), "loc_fts": (1,), "nav_types": (1,), "view_lens": ()},
    "navigation": {"txt_embeds": (1,), "txt_masks": (1,), "gmap_step_ids": (1,), "gmap_img_fts": (1,),
                   "gmap_pos_fts": (1,), "gmap_masks": (1,), "gmap_visited_masks": (1,), "gmap_pair_dists": (1, 2),
                   "bev_fts": (), "bev_pos_fts": (), "bev_masks": (), "bev_nav_masks": (), "bev_cand_idxs": (1,)},
}


def ce_nav_bucket(mode, batch):
    """nav_bucket of the CE calls: B exact (the CE rollout drops finished episodes), every other length rounded to 8"""
    return _bucket(CE_NAV_PAD_DIMS, mode, batch)


def ce_nav_pad(mode, batch, device):
    return _pad(CE_NAV_PAD_DIMS, mode, batch, device)


def ce_nav_eager(model, mode, batch):
    """the network's own method (not an instance attribute that routes to a replay)"""
    name = _CE_METHOD[mode]
    return getattr(type(model), name)(model, *[batch[k] for k in CE_NAV_CALLS[name][1]])


def ce_nav_forward_padded(model, mode, pad, host=None):
    """the CE network on padded inputs `pad` (ce_nav_pad); `host` as for nav_forward_padded"""
    if mode == "panorama":
        return type(model).forward_panorama(model, *[pad.get(k) for k in CE_NAV_CALLS["forward_panorama"][1]],
                                            vtot=pad["loc_fts"].shape[1])
    if mode == "navigation":
        pad = dict(pad, gmap_vpids=host[0], bev_cand_vpids=host[1])
    return ce_nav_eager(model, mode, pad)


def ce_nav_slice(mode, out, batch):
    if mode != "navigation":
        return nav_slice(mode, out, batch)
    c = torch.Tensor.clone
    G, Kc = batch["gmap_masks"].shape[1], batch["bev_cand_idxs"].shape[1]
    return {"gmap_embeds": c(out["gmap_embeds"][:, :G]), "global_logits": c(out["global_logits"][:, :G]),
            "local_logits": c(out["local_logits"][:, :Kc]), "fused_logits": c(out["fused_logits"][:, :G])}


CE_NAV = Surface(CE_NAV_PAD_DIMS, ce_nav_forward_padded, ce_nav_slice, ce_nav_eager)


def install_ce_replay(net):
    """Routes the CE network's `forward_txt` / `forward_panorama` / `forward_navigation` through a GraphedNavigation
    over the CE surface: eval-mode calls under torch.no_grad() replay graphs of padded shape buckets, every other call
    runs the network's own method.  The module, its state_dict and its train / eval switch are unchanged.  Install on
    the policy's network (`policy.net.vln_bert`); -> the GraphedNavigation (its `launches`, `entries`)."""
    replay = GraphedNavigation(net, CE_NAV)
    for name, (mode, args) in CE_NAV_CALLS.items():
        def call(*a, _mode=mode, _args=args, **kw):
            batch = dict(zip(_args, a))
            batch.update(kw)
            return replay(_mode, batch)
        setattr(net, name, call)
    return replay


# ------------------------------------------------------------------- VLN-CE policy RGB encoder (model/clip_visual.py)
# One mode; the input is observations["rgb"] at its exact shape (N = 12 views x B environments) and dtype.
CE_RGB_DIMS = {"rgb": {"rgb": ()}}
CE_RGB = Surface(CE_RGB_DIMS, lambda tower, mode, pad, host=None: tower.encode_rgb(pad["rgb"]),
                 lambda mode, out, batch: (out[0].clone(), out[1].clone()),
                 lambda tower, mode, batch: tower.encode_rgb(batch["rgb"]),
                 grad_ok=True, stale=lambda tower: tower.changed())


def install_ce_rgb_encoder(rgb_encoder):
    """Routes the CE policy's `CLIPEncoderB16` instance (`policy.net.rgb_encoder`, `policy.net.module.rgb_encoder`
    with data parallelism) to the kernels: `rgb_encoder(observations)` returns (rgb_vector, rgb_grid) as fresh fp32
    tensors, computed by model.clip_visual.ClipTower from the weights of `rgb_encoder.model.visual` with the mean / std
    of its `rgb_transform`.  While the encoder is in eval mode every call, with or without grad, replays the CUDA graph
    of its image count N (one graph per N; N = 12 B shrinks as episodes finish) on a static copy of
    observations["rgb"]; in training mode, or if a capture fails, the same kernels run eagerly.  A weight change
    (load_state_dict) is seen by the next call either way.  The module, the policy's state_dict, checkpoints and the
    train / eval switch are unchanged.  -> the GraphedNavigation (its `launches`, `entries`)."""
    from .model.clip_visual import ClipTower
    norm = rgb_encoder.rgb_transform[-1]
    tower = ClipTower(rgb_encoder.model.visual, mean=norm.mean, std=norm.std, owner=rgb_encoder)
    replay = GraphedNavigation(tower, CE_RGB)

    def forward(observations):
        tower.check_grad()
        return replay("rgb", {"rgb": observations["rgb"]})
    rgb_encoder.forward = forward
    return replay


# ------------------------------------------------------------------------ VLN-CE waypoint predictor (model/waypoint.py)
# One mode; the input is the depth features at their exact shape (N = 12 views x B environments) and dtype.  rgb_feats
# only decides B, which the depth features' N repeats, so it is not copied into the graph's buffers.
CE_WAYPOINT_DIMS = {"waypoint": {"depth_feats": ()}}
CE_WAYPOINT = Surface(CE_WAYPOINT_DIMS, lambda runner, mode, pad, host=None: runner.logits(pad["depth_feats"]),
                      lambda mode, out, batch: out.clone(),
                      lambda runner, mode, batch: runner.logits(batch["depth_feats"]),
                      grad_ok=True, stale=lambda runner: runner.changed())


def install_ce_waypoint_predictor(waypoint_predictor):
    """Routes the trainer's waypoint predictor (TRM_net.py BinaryDistPredictor_TRM; under nn.DataParallel the wrapped
    `.module`) to the kernels: `waypoint_predictor(rgb_feats, depth_feats)` returns the heatmap logits (B, 120, 12) as
    a fresh fp32 tensor, computed by model.waypoint.WaypointRunner from the module's own weights.  Every eval-mode call,
    with or without grad (the trainer freezes the predictor), replays the CUDA graph of its view count N (one graph per
    N = 12 B) on a static copy of depth_feats; a capture that fails runs the same kernels eagerly.  A call in training
    mode, or with grad enabled while a parameter requires grad, raises.  A weight change (load_state_dict) is seen by
    the next call.  The module, its state_dict and its train / eval switch are unchanged.  -> the GraphedNavigation
    (its `launches`, `entries`)."""
    from .model.waypoint import WaypointRunner
    module = waypoint_predictor
    if isinstance(module, (torch.nn.DataParallel, torch.nn.parallel.DistributedDataParallel)):
        module = module.module
    runner = WaypointRunner(module)
    replay = GraphedNavigation(runner, CE_WAYPOINT)

    def forward(rgb_feats, depth_feats):
        runner.check_call()
        return replay("waypoint", {"depth_feats": runner.check_inputs(rgb_feats, depth_feats)})
    module.forward = forward
    return replay


# ------------------------------------------------------------------ VLN-CE policy depth encoder (model/depth_resnet.py)
# One mode; the input is observations["depth"] at its exact shape (N = 12 views x B environments) and dtype.
CE_DEPTH_DIMS = {"depth": {"depth": ()}}
CE_DEPTH = Surface(CE_DEPTH_DIMS, lambda tower, mode, pad, host=None: tower.encode(pad["depth"]),
                   lambda mode, out, batch: out.clone(),
                   lambda tower, mode, batch: tower.encode(batch["depth"]),
                   grad_ok=True, stale=lambda tower: tower.changed())


def install_ce_depth_encoder(depth_encoder):
    """Routes the CE policy's `VlnResnetDepthEncoder` instance (`policy.net.depth_encoder`,
    `policy.net.module.depth_encoder` with data parallelism) to the kernels: its `visual_encoder(observations)` returns
    the (N, 128, 4, 4) features as a fresh fp32 tensor, computed by model.depth_resnet.DepthTower from the weights of
    `depth_encoder.visual_encoder`, so the wrapper's own `depth_features` and `spatial_output` branches are unchanged.
    While the encoder is in eval mode every call, with or without grad, replays the CUDA graph of its image count N (one
    graph per N; N = 12 B shrinks as episodes finish) on a static copy of observations["depth"]; in training mode, or if
    a capture fails, the same kernels run eagerly.  A call with grad enabled while an encoder parameter requires grad
    (trainable=True) raises.  A weight change (load_state_dict) is seen by the next call either way.  The module, the
    policy's state_dict, checkpoints and the train / eval switch are unchanged.  -> the GraphedNavigation (its
    `launches`, `entries`)."""
    from .model.depth_resnet import DepthTower
    visual = depth_encoder.visual_encoder
    tower = DepthTower(visual, owner=depth_encoder)
    replay = GraphedNavigation(tower, CE_DEPTH)

    def forward(observations):
        tower.check_grad()
        return replay("depth", {"depth": observations["depth"]})
    visual.forward = forward
    return replay


# ------------------------------------------------------------ VLN-CE policy `waypoint` call (model/ce_waypoint_step.py)
# One mode; the only input is the (24, 5) view table, staged on the device before each call.  The geometry (B, rgb and
# depth image sizes) and in_train are the call's shape key, so training and eval rollouts keep a graph each.
CE_STEP_DIMS = {"waypoint": {"views": ()}}
_WAYPOINT_ARGS = ("mode", "waypoint_predictor", "observations", "in_train")


def install_ce_waypoint_step(net, waypoint_aug=False):
    """Makes the CE policy network's `waypoint` call (Policy_ViewSelection_BEV.py BEV.forward with mode='waypoint')
    one CUDA graph replay: install on `policy.net` (`policy.net.module` under DDP); `net.forward` is replaced.  A call
    with mode='waypoint' and in_train=False whose observations model.ce_waypoint_step.covered accepts runs
    model.ce_waypoint_step.WaypointStep over the network's encoders and the call's `waypoint_predictor` (unwrapped
    from DataParallel; a different predictor module rebuilds the step's graphs), replaying one graph per (B, image
    sizes, in_train) whatever the network's train / eval switch, and returns the reference's output dict (a
    StepOutputs).  With waypoint_aug=True, covered in_train=True calls (the trainer's IL.waypoint_aug rollouts) are the
    step's too: each replay draws fresh Exp(1) noise from torch's default CUDA generator and samples every candidate
    from it, with the reference's distribution and algorithm but not its random stream.  Every other call (other
    modes, in_train=True unless waypoint_aug, observations not covered) runs the original forward unchanged.  A weight
    change (load_state_dict) of any of the three modules is seen by the next call.  -> the WaypointStep (its `replay`,
    a GraphedNavigation, once a call has been replayed)."""
    import inspect
    from .model import ce_waypoint_step as CS
    step = CS.WaypointStep(net)
    step.replay = None
    original = net.forward
    sig = inspect.signature(original)

    # the shape key (B, Hr, Wr, Hd, Wd, in_train) reaches `padded` as `host`
    def eager(st, mode, batch):                 # a bucket without a graph: the same kernels and the same output dict
        return st.outputs(st.run(batch["views"], batch["geom"], batch["in_train"]), batch["geom"][0])
    surface = Surface(CE_STEP_DIMS, lambda st, mode, pad, host=None: st.run(pad["views"], host[:5], host[5]),
                      lambda mode, out, batch: step.outputs(out, batch["geom"][0]), eager,
                      grad_ok=True, stale=lambda st: st.changed(),
                      shape_key=lambda mode, batch: batch["geom"] + (batch["in_train"],))

    def forward(*args, **kwargs):
        bound = sig.bind(*args, **kwargs)
        bound.apply_defaults()
        a = bound.arguments
        if (a["mode"] != "waypoint" or (a["in_train"] and not waypoint_aug)
                or not isinstance(a["observations"], dict)):
            return original(*args, **kwargs)
        cov = CS.covered(a["observations"], step.clip.res, step.device)
        if cov is None:
            return original(*args, **kwargs)
        if step.set_predictor(a["waypoint_predictor"]):
            step.replay = GraphedNavigation(step, surface)
        step.check_call()
        pairs, geom = cov
        table = CS.view_table(a["observations"], pairs).pin_memory().to(step.device, non_blocking=True)
        return step.replay("waypoint", {"views": table, "geom": geom, "in_train": bool(a["in_train"])})
    net.forward = forward
    return step


def install_ce_vp_features(trainer):
    """Replaces the CE trainer's `_vp_feature_variable(obs)`: for outputs of an installed waypoint step
    (install_ce_waypoint_step) it returns the step's padded panorama inputs, sliced to the batch's longest view list,
    with loc_fts, nav_types and view_lens built on the host and uploaded in one copy; any other dict goes to the
    trainer's original method."""
    from .model.ce_waypoint_step import StepOutputs
    original = trainer._vp_feature_variable

    def vp_feature_variable(obs):
        if isinstance(obs, StepOutputs):
            return obs.vp_inputs()
        return original(obs)
    trainer._vp_feature_variable = vp_feature_variable
    return vp_feature_variable


def install_ce_gmap_features(trainer):
    """Builds the CE trainer's `gmap_img_fts` on the kernels (ce_gmap.py) instead of the rollout's per-environment
    tensor glue.  On the trainer's instances only:
      * `trainer.policy.net`'s `panorama` calls record their outputs (pano_embeds, the call's nav_types, pano_masks) in
        the episode's ce_gmap.Memory, which starts when the call first sees a fresh `trainer.gmaps`;
      * each of those GraphMaps gets an `update_graph` that replaces the embedding arguments the rollout passes with
        handles to the step's rows (ghost merges add handles, in merge order) before running the original, and a
        `get_node_embeds` that returns the row the kernel computes, so other callers keep working;
      * `trainer._nav_gmap_variable` runs the trainer's own method for every other key and returns `gmap_img_fts`
        from one bb_ce_gmap_features launch, differentiable with respect to every stored step's pano_embeds.
    Nothing in it synchronises with the host.  The rollout's own masked mean and boolean index still run, and their
    results are no longer read.  -> the installed _nav_gmap_variable."""
    from . import ce_gmap
    net, original = trainer.policy.net, trainer._nav_gmap_variable
    forward = net.forward

    @functools.wraps(forward)       # keeps the signature, which install_ce_waypoint_step binds, if installed after this
    def panorama_forward(*args, **kwargs):
        out = forward(*args, **kwargs)
        if kwargs.get("mode") == "panorama":
            mem = ce_gmap.episode(trainer.gmaps)
            if mem is None:
                mem = ce_gmap.Memory()
                for g in trainer.gmaps:
                    ce_gmap.attach(trainer, g, mem)
            mem.record(out[0], kwargs["nav_types"], out[1])
        return out

    def nav_gmap_variable(cur_vp, cur_pos, cur_ori):
        out, rows = ce_gmap.trainer_method(original, trainer.gmaps, cur_vp, cur_pos, cur_ori)
        out["gmap_img_fts"] = ce_gmap.episode(trainer.gmaps).features(rows)
        return out
    net.forward = panorama_forward
    trainer._nav_gmap_variable = nav_gmap_variable
    return nav_gmap_variable


def install_ce_lift(trainer):
    """Replaces the CE trainer's `lift(cur_pos, cur_ori, rgb_grid, depth_grid)` with agent_bev.ce_lift: the heading fan
    in one upload and PointCloud.forward in one bb_bev_lift_points launch, with no host synchronisation.  The projector
    is checked here (ValueError if the kernel does not reproduce it) and again on every call.  update_node_pc,
    gather_node_pc and _nav_bev_variable read the clouds as before.  -> the installed lift."""
    from . import agent_bev
    agent_bev.lift_intrinsics(trainer.projector)

    def lift(cur_pos, cur_ori, rgb_grid, depth_grid):
        return agent_bev.ce_lift(trainer, cur_pos, cur_ori, rgb_grid, depth_grid)
    trainer.lift = lift
    return lift


class GraphedNavigation:
    """The agents' per-step calls `model(mode, batch)` (GlocalTextPathNavCMT: language / panorama / navigation) replayed
    as CUDA graphs.  Called like the model, with the same inputs and outputs.

    In eval mode under torch.no_grad() each call copies its inputs into the static buffers of its shape bucket
    (`nav_bucket`: every variable length rounded up to a multiple of 8, zero padding) and replays the bucket's graph,
    captured at its first call; outputs are sliced back to the caller's shapes as fresh tensors (the agents keep views
    of them across steps, which a view of a static buffer would not survive).  The SAP fusion matches are host string
    work: they are written into the bucket's pinned staging buffer before the replay, and the graph's copy node reads
    them from there.  Training or grad-enabled calls (DAgger rollouts), and buckets whose capture failed, run the model
    eagerly and unchanged.

    Weights: a replay reads the bf16 weight shadows without `WeightCache.get`, so they are all re-cast in place (one
    launch, `refresh_all`) at every `language` call -- once per episode -- and before the first replay.  That picks up
    `load_state_dict` and optimizer steps between validations.  A parameter whose storage moved since a graph was
    captured (`.to()`, the packed-bias re-homing of `WeightCache.vec`) drops that graph; it is captured again at its
    next call.  All graphs share one memory pool.  With G <= 100 map nodes there are at most 13 G-buckets per (B,
    K-bucket).

    Agent side: `vln_bert.vln_bert.forward = GraphedNavigation(vln_bert.vln_bert)` keeps the module, its state_dict and
    its train / eval switch, and routes its calls here.  `surface` names the per-step API (NAV, the agents'
    `forward(mode, batch)`; CE_NAV, the CE policy's three methods, installed by `install_ce_replay`)."""

    def __init__(self, model, surface=NAV):
        self.model, self.s = model, surface
        self.params = list(model.parameters())
        self.entries = {}
        self.pool = None
        self.fresh = False

    def _eager(self, mode, batch):
        return self.s.eager(self.model, mode, batch)

    def _param_ptrs(self):
        return tuple(p.data_ptr() for p in self.params)

    def refresh(self):
        """Re-cast every weight shadow from the current parameters and drop graphs whose parameters moved."""
        self.model.rt.wc.refresh_all(padded=True)
        ptrs = self._param_ptrs()
        for k in [k for k, e in self.entries.items() if e.get("ptrs") not in (None, ptrs)]:
            ent = self.entries.pop(k)
            if ent["stage"] is not None:
                ent["done"].synchronize()   # its last replay may still have to copy the pinned staging buffer
        self.fresh = True

    def __call__(self, mode, batch):
        if self.model.training or (torch.is_grad_enabled() and not self.s.grad_ok) or mode not in self.s.dims:
            return self._eager(mode, batch)
        if mode == "language" or not self.fresh or (self.s.stale is not None and self.s.stale(self.model)):
            self.refresh()
        key = self._key(mode, batch)
        ent = self.entries.get(key)
        if ent is None:
            ent = self.entries[key] = self._new_entry(mode, batch)
        if ent["failed"]:
            return self._eager(mode, batch)
        self._fill(ent, mode, batch)
        if ent["graph"] is None:
            try:
                self._capture(ent, mode)
            except Exception as e:          # e.g. a host synchronisation inside forward: this bucket stays eager
                import warnings
                warnings.warn("CUDA-graph capture of the %s call failed (%s: %s); running it eagerly" % (
                    mode, type(e).__name__, str(e)[:200]))
                torch.cuda.synchronize()
                ent["failed"] = True
                return self._eager(mode, batch)
        ent["graph"].replay()
        if ent["stage"] is not None:
            ent["done"].record()
        return self.s.slice(mode, ent["out"], batch)

    def _key(self, mode, batch):
        key = _bucket(self.s.dims, mode, batch)
        return key if self.s.shape_key is None else key + (self.s.shape_key(mode, batch),)

    def _new_entry(self, mode, batch):
        dev = self.params[0].device
        bufs = {}
        for name, k in zip(self.s.dims[mode], _bucket(self.s.dims, mode, batch)[2:]):
            if k is not None:
                bufs[name] = torch.zeros(k[0], dtype=k[1], device=dev)
        ent = {"in": bufs, "ext": {}, "graph": None, "out": None, "failed": False, "ptrs": None, "launches": None,
               "stage": None, "host": None if self.s.shape_key is None else self.s.shape_key(mode, batch)}
        if mode == "navigation":
            B, G = bufs["gmap_masks"].shape
            Kc = bufs["bev_cand_idxs"].shape[1]
            ent["stage"] = torch.zeros(2, B, G, Kc, dtype=torch.float32, pin_memory=True)
            ent["done"] = torch.cuda.Event()
        return ent

    def _fill(self, ent, mode, batch):
        for name, buf in ent["in"].items():
            x = batch[name]
            ext, last = tuple(x.shape), ent["ext"].get(name)
            if last is not None and any(a < b for a, b in zip(ext, last)):
                buf.zero_()                 # the previous call of this bucket left real values beyond the new extent
            buf[tuple(slice(0, n) for n in ext)].copy_(x)
            ent["ext"][name] = ext
        if ent["stage"] is not None:
            # the previous replay of this bucket must have copied the staging buffer before the host rewrites it
            if ent["graph"] is not None:
                ent["done"].synchronize()
            _, B, G, Kc = ent["stage"].shape
            gv = ops.PreparedList(batch["gmap_vpids"])
            cands = batch["bev_cand_vpids"]
            ops._fusion_matches(gv, [c[1:] for c in cands], G, Kc, out=ent["stage"])
            gv.host_fusion = ((G, Kc), ent["stage"])
            ent["host"] = (gv, cands)

    def _capture(self, ent, mode):
        torch.cuda.synchronize()
        # eager warm-up on the static buffers: weight shadows, packed biases, library workspaces, cuBLAS state
        self.s.padded(self.model, mode, ent["in"], ent["host"])
        torch.cuda.synchronize()
        if self.pool is None:
            self.pool = torch.cuda.graph_pool_handle()
        g = torch.cuda.CUDAGraph()
        n0 = K.launch_count()
        with torch.cuda.graph(g, pool=self.pool):
            out = self.s.padded(self.model, mode, ent["in"], ent["host"])
        ent["launches"] = K.launch_count() - n0
        ent["graph"], ent["out"], ent["ptrs"] = g, out, self._param_ptrs()

    def launches(self, mode, batch):
        """kernels of libbevbert_b200.so inside the graph of this call's bucket, or None when it runs eagerly."""
        ent = self.entries.get(self._key(mode, batch))
        return ent["launches"] if ent is not None and ent["graph"] is not None else None
