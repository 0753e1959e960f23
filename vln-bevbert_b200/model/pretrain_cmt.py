"""GlocalTextPathCMTPreTraining on the H100 kernels -- drop-in for pretrain_src/model/pretrain_cmt.py.

`forward(batch, task, compute_loss=True)` has the reference's contract (pretrain_cmt.py:169-238): it takes
the collated batch dict, runs the BEV
lift-splat, the hybrid-map encoder and the task head, and returns the per-item loss tensor (or the logits
tuple).  Requires CUDA tensors -- there is no CPU path.
"""
from collections import defaultdict
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import blocks as Bk
from .bev_utils import PointCloud, bevpos_polar
from .ops import build_sap_fusion, gen_seq_masks
from .vilmodel import BertLayerNorm, BertOnlyMLMHead, GlocalTextPathCMT, PreTrainedBase

BEV_DIM = 21
BEV_RES = 0.5


def build_projector(bev_dim=None, bev_res=None, device=None):
    """pretrain_cmt.py:19-32: projector for 14x14 patch grids with a 90 deg vfov + the polar BEV position code."""
    D = BEV_DIM if bev_dim is None else bev_dim
    res = BEV_RES if bev_res is None else bev_res
    projector = PointCloud(math.radians(90), 1, feature_map_height=14, feature_map_width=14, map_dim=D, map_res=res,
                           z_clip_threshold=0.5)
    bev_pos = bevpos_polar(D).reshape(D * D, 3)[None, :, :]
    return projector, (bev_pos.to(device) if device is not None else bev_pos)


class _Head(nn.Module):
    """Linear -> ReLU -> LN(1e-12) -> Linear (RegionClassification / ClsPrediction / MulClsPrediction,
    pretrain_cmt.py:34-71); parameters live in `net` with the reference's indices 0, 2, 3."""

    def __init__(self, hidden_size, out_dim, input_size=None):
        super().__init__()
        input_size = hidden_size if input_size is None else input_size
        self.net = nn.Sequential(nn.Linear(input_size, hidden_size), nn.ReLU(), BertLayerNorm(hidden_size, eps=1e-12),
                                 nn.Linear(hidden_size, out_dim))

    def forward(self, rt, x):
        n = self.net
        return Bk.run_block(Bk.HeadImpl(rt), [x], [n[0].weight, n[0].bias, n[2].weight, n[2].bias, n[3].weight, n[3].bias])


class RegionClassification(_Head):
    def __init__(self, hidden_size, label_dim):
        super().__init__(hidden_size, label_dim)


class ClsPrediction(_Head):
    def __init__(self, hidden_size, input_size=None):
        super().__init__(hidden_size, 1, input_size)


class MulClsPrediction(_Head):
    def __init__(self, hidden_size, input_size=None):
        super().__init__(hidden_size, 40, input_size)


class GlocalTextPathCMTPreTraining(PreTrainedBase):
    def __init__(self, config):
        super().__init__(config)
        self.bert = GlocalTextPathCMT(config)
        self.bert._rt_external = True
        self.rt = self.bert.rt
        self.drop_env = nn.Dropout(config.feat_dropout)
        h = config.hidden_size
        if "mlm" in config.pretrain_tasks:
            self.mlm_head = BertOnlyMLMHead(config)
        if "mrc" in config.pretrain_tasks:
            self.obj_classifier = RegionClassification(h, config.obj_prob_size)
        if "sap" in config.pretrain_tasks:
            self.global_sap_head = ClsPrediction(h)
            self.local_sap_head = ClsPrediction(h)
            self.sap_fuse_linear = ClsPrediction(h, input_size=h * 2) if config.glocal_fuse else None
        if "og" in config.pretrain_tasks:
            self.og_head = ClsPrediction(h)
        if "sem" in config.pretrain_tasks or "masksem" in config.pretrain_tasks:
            self.local_sem_head = MulClsPrediction(h)
            self.sem_pred_token = config.sem_pred_token
        self.init_weights()
        self.tie_weights()
        self.bev_res = getattr(config, "bev_res", BEV_RES)
        self.projector, self.bev_pos_fts = build_projector(config.bev_dim, self.bev_res)

    def tie_weights(self):  # pretrain_cmt.py:109-112
        if "mlm" in self.config.pretrain_tasks:
            self.mlm_head.predictions.decoder.weight = self.bert.embeddings.word_embeddings.weight

    # ------------------------------------------------------------------------------------------ BEV lift-splat
    @torch.no_grad()
    def lift_splat(self, batch):
        """pretrain_cmt.py:114-167 on the fused kernels: cell index straight from depth + poses, then the
        deterministic scatter-mean of the patch features / semantic labels."""
        rgbs, depths, sems = batch.pop("rgbs"), batch.pop("depths"), batch.pop("sems")
        T_c2w, T_w2c, S_w2c = batch.pop("T_c2w"), batch.pop("T_w2c"), batch.pop("S_w2c")
        gpos = batch.pop("bev_gpos_fts")
        bs = rgbs.shape[0]
        D = self.config.bev_dim
        idx, _ = self.projector.lift_index(depths, T_c2w, S_w2c, T_w2c, depth_scale=10.0)
        # sems: float64 one-hots (B, 2352, 40) as collated by the reference, or the uint8 class ids (B, 2352) they were
        # expanded from (ops.prepare_batch wire format)
        sems = sems.reshape(bs, -1) if sems.dtype == torch.uint8 else sems.reshape(bs, -1, sems.shape[-1])
        bev, _, ob, bsem, bsem_mask = self.projector.splat(idx, rgbs.reshape(bs, -1, rgbs.shape[-1]), sems)
        if self.bev_pos_fts.device != bev.device:
            self.bev_pos_fts = self.bev_pos_fts.to(bev.device)
        pos = torch.cat([gpos.expand(-1, D * D, -1), self.bev_pos_fts.expand(bs, -1, -1)], dim=-1)
        batch.update({"bev_fts": bev, "bev_masks": torch.ones(bs, D * D, dtype=torch.bool, device=bev.device),
                      "bev_pos_fts": pos, "bev_sems": bsem, "bev_sem_masks": bsem_mask, "bev_ob_masks": ob,
                      "bev_cell_idx": idx})
        return batch

    def drop_feats(self, batch):
        """The reference applies nn.Dropout to the fp32 features here (pretrain_cmt.py:102-106); we record the
        probability and apply it inside the fp32->bf16 cast that feeds the first GEMM of each feature stream."""
        self.rt.feat_p = self.drop_env.p if self.training else 0.0
        return batch

    # ------------------------------------------------------------------------------------------ dispatch
    _BERT_KEYS = ("txt_ids", "txt_lens", "traj_view_img_fts", "traj_obj_img_fts", "traj_loc_fts", "traj_nav_types",
                  "traj_step_lens", "traj_vp_view_lens", "traj_vp_obj_lens", "traj_vpids", "traj_cand_vpids",
                  "gmap_lens", "gmap_step_ids", "gmap_pos_fts", "gmap_pair_dists", "gmap_vpids", "bev_fts",
                  "bev_pos_fts", "bev_masks", "bev_nav_masks")

    def forward(self, batch, task, compute_loss=True):
        batch = defaultdict(lambda: None, batch)   # a copy: the caller's dict is left untouched, as in the reference
        self.rt.begin(self.training, tag=task)
        batch = self.lift_splat(batch)
        batch = self.drop_feats(batch)
        args = [batch[k] for k in self._BERT_KEYS]
        if task.startswith("mlm"):
            return self.forward_mlm(*args, batch["txt_labels"], compute_loss)
        if task.startswith("mrc"):
            return self.forward_mrc(*args, batch["vp_obj_mrc_masks"], batch["vp_obj_probs"], compute_loss)
        if task.startswith("sap"):
            return self.forward_sap(*args[:16], batch["gmap_visited_masks"], *args[16:], batch["bev_cand_idxs"],
                                    batch["global_act_labels"], batch["local_act_labels"], compute_loss)
        if task.startswith("og"):
            return self.forward_og(*args, batch["obj_labels"], compute_loss)
        if task.startswith("sem"):
            return self.forward_sem(*args, batch["bev_sems"], batch["bev_sem_masks"], compute_loss)
        if task.startswith("masksem"):
            return self.forward_masksem(*args, batch["bev_sems"], batch["bev_sem_masks"], batch["bev_mrc_masks"],
                                        compute_loss)
        raise ValueError("invalid task")

    def _masked_rows(self, hidden, mask):
        """rows of (B,n,H) `hidden` where bool (B,n) `mask` (pretrain_cmt.py:266-270), via the gather kernel."""
        idx = torch.nonzero(mask.reshape(-1), as_tuple=False).reshape(-1)
        return Bk.run_block(Bk.GatherRowsImpl(), [hidden.reshape(-1, hidden.shape[-1]), idx], [])

    # ------------------------------------------------------------------------------------------ tasks
    def forward_mlm(self, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                    traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens,
                    gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks,
                    bev_nav_masks, txt_labels, compute_loss):
        txt_embeds = self.bert.forward_mlm(
            txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types, traj_step_lens,
            traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens, gmap_step_ids, gmap_pos_fts,
            gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks)
        return self._mlm_head(txt_embeds, gmap_vpids, txt_labels, compute_loss)

    def _mlm_head(self, txt_embeds, gmap_vpids, txt_labels, compute_loss):
        """pretrain_cmt.py:217-227: MLM scores / loss of the masked text rows."""
        impl = Bk.MLMLossImpl(self.rt, self.mlm_head.eps, compute_loss)
        pre = getattr(gmap_vpids, "host_mlm", None)      # ops.prepare_batch(): masked rows listed at collate time
        if pre is not None and pre[0] == tuple(txt_labels.shape):
            dev = txt_embeds.device
            idx, labels = pre[1].to(dev, non_blocking=True), pre[2].to(dev, non_blocking=True)
            masked_output = Bk.run_block(Bk.GatherRowsImpl(), [txt_embeds.reshape(-1, txt_embeds.shape[-1]), idx], [])
            return Bk.run_block(impl, [masked_output, labels], self.mlm_head.params())
        sel = txt_labels != -1
        masked_output = self._masked_rows(txt_embeds, sel)
        return Bk.run_block(impl, [masked_output, txt_labels[sel]], self.mlm_head.params())

    def forward_mrc(self, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                    traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens,
                    gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks,
                    bev_nav_masks, vp_obj_mrc_masks, vp_obj_probs, compute_loss=True):
        _, _, obj_embeds, _ = self.bert(
            txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types, traj_step_lens,
            traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens, gmap_step_ids, gmap_pos_fts,
            gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks, return_gmap_embeds=False)
        logits = self.obj_classifier(self.rt, self._masked_rows(obj_embeds, vp_obj_mrc_masks))
        targets = vp_obj_probs[vp_obj_mrc_masks]
        if not compute_loss:
            return logits, targets
        return F.kl_div(F.log_softmax(logits, dim=-1), targets, reduction="none").sum(dim=1)

    def forward_sap(self, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                    traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens,
                    gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, gmap_visited_masks, bev_fts, bev_pos_fts,
                    bev_masks, bev_nav_masks, bev_cand_idxs, global_act_labels, local_act_labels, compute_loss):
        gmap_embeds, bev_embeds, _, _ = self.bert(
            txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types, traj_step_lens,
            traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens, gmap_step_ids, gmap_pos_fts,
            gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks)
        return self._sap_head(gmap_embeds, bev_embeds, traj_cand_vpids, gmap_lens, gmap_vpids, gmap_visited_masks,
                              bev_nav_masks, bev_cand_idxs, global_act_labels, local_act_labels, compute_loss)

    def _sap_head(self, gmap_embeds, bev_embeds, traj_cand_vpids, gmap_lens, gmap_vpids, gmap_visited_masks,
                  bev_nav_masks, bev_cand_idxs, global_act_labels, local_act_labels, compute_loss):
        """pretrain_cmt.py:322-366: global / local / fused action logits and their losses."""
        B = gmap_embeds.shape[0]
        G, Kc = gmap_embeds.shape[1], bev_cand_idxs.shape[1]
        n = self.config.bev_dim * self.config.bev_dim
        dev = gmap_embeds.device
        bev_flat = bev_embeds.reshape(-1, bev_embeds.shape[-1]) if bev_embeds.is_contiguous() else \
            bev_embeds.contiguous().view(-1, bev_embeds.shape[-1])
        base = torch.arange(B, device=dev)[:, None] * n
        cand_embeds = Bk.run_block(Bk.GatherRowsImpl(), [bev_flat, (base + bev_cand_idxs).reshape(-1)], [])
        cand_masks = bev_nav_masks[torch.arange(B, device=dev)[:, None], bev_cand_idxs]
        if self.sap_fuse_linear is None:
            fuse = 0.5
        else:
            centre = (n - 1) // 2
            g0 = Bk.run_block(Bk.GatherRowsImpl(), [gmap_embeds.reshape(-1, gmap_embeds.shape[-1]),
                                                    torch.arange(B, device=dev) * G], [])
            c0 = Bk.run_block(Bk.GatherRowsImpl(), [bev_flat, torch.arange(B, device=dev) * n + centre], [])
            fuse = torch.sigmoid(self.sap_fuse_linear(self.rt, torch.cat([g0, c0], 1)))          # (B,1) fp32
        global_logits = self.global_sap_head(self.rt, gmap_embeds).squeeze(2) * fuse
        global_logits = global_logits.masked_fill(gmap_visited_masks, -float("inf"))
        global_logits = global_logits.masked_fill(gen_seq_masks(gmap_lens, G).logical_not(), -float("inf"))
        local_logits = self.local_sap_head(self.rt, cand_embeds).view(B, Kc) * (1 - fuse)
        local_logits = local_logits.masked_fill(cand_masks.logical_not(), -float("inf"))
        # fusion (pretrain_cmt.py:339-356) through a host-built 0/1 matrix; -inf candidates are never selected
        Fm = build_sap_fusion(gmap_vpids, gmap_visited_masks, [c[-1] for c in traj_cand_vpids], G, Kc, dev)
        local_fin = local_logits.masked_fill(cand_masks.logical_not(), 0.0)
        fused_logits = global_logits + torch.einsum("bgk,bk->bg", Fm, local_fin)
        # keep the -inf semantics of `fused[:, 0] += local[:, 0]` (no host sync: unconditional select)
        fused_logits = torch.cat([torch.where(torch.isinf(local_logits[:, :1]), local_logits[:, :1], fused_logits[:, :1]),
                                  fused_logits[:, 1:]], 1)
        if not compute_loss:
            return global_logits, local_logits, fused_logits, global_act_labels, local_act_labels
        return F.cross_entropy(global_logits, global_act_labels, reduction="none") + \
            F.cross_entropy(local_logits, local_act_labels, reduction="none") + \
            F.cross_entropy(fused_logits, global_act_labels, reduction="none")

    def forward_og(self, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                   traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens,
                   gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks,
                   bev_nav_masks, obj_labels, compute_loss):
        _, _, obj_embeds, obj_masks = self.bert(
            txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types, traj_step_lens,
            traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens, gmap_step_ids, gmap_pos_fts,
            gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks, return_gmap_embeds=False)
        obj_logits = self.og_head(self.rt, obj_embeds.contiguous()).squeeze(2)
        obj_logits = obj_logits.masked_fill(obj_masks.logical_not(), -float("inf"))
        return F.cross_entropy(obj_logits, obj_labels, reduction="none") if compute_loss else obj_logits

    # sync_free_mean = True (set by graphs.GraphedTrainStep): sem / masksem return the MEAN of the per-item loss as a
    # 0-d tensor, computed over all cells with the selection as a weight -- the number of labelled cells is known only
    # on the device (lift_splat computes bev_sem_masks there), so the reference's variable-length (n_cells, 40) result
    # would need a device->host synchronisation and could not live in a CUDA graph.  Same value and gradients as
    # `forward(...).mean()`.
    sync_free_mean = False

    def _sem(self, args, bev_sems, sel, compute_loss):
        bev_embeds = self.bert.forward_sem(*args, sem_pred_token=self.sem_pred_token)
        if self.sync_free_mean and compute_loss:
            logits = self.local_sem_head(self.rt, bev_embeds.reshape(-1, bev_embeds.shape[-1]))
            per = F.binary_cross_entropy_with_logits(logits, bev_sems.reshape(-1, bev_sems.shape[-1]).float(), reduction="none")
            w = sel.reshape(-1, 1).to(per.dtype)
            return (per * w).sum() / (w.sum() * per.shape[1])
        sem_logits = self.local_sem_head(self.rt, self._masked_rows(bev_embeds, sel))
        sem_labels = bev_sems[sel].float()
        if not compute_loss:
            return sem_logits, sem_labels
        return F.binary_cross_entropy_with_logits(sem_logits, sem_labels, reduction="none")

    def forward_sem(self, *a):
        *args, bev_sems, bev_sem_masks, compute_loss = a
        return self._sem(args, bev_sems, bev_sem_masks, compute_loss)

    def forward_masksem(self, *a):
        *args, bev_sems, bev_sem_masks, bev_mrc_masks, compute_loss = a
        args = list(args)
        args[16] = args[16].masked_fill(bev_mrc_masks.unsqueeze(-1), 0)      # bev_fts (pretrain_cmt.py:423-424)
        return self._sem(args, bev_sems, bev_sem_masks & bev_mrc_masks, compute_loss)
