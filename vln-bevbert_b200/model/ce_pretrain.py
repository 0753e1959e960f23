"""The VLN-CE pre-training model on the H100 kernels -- drop-in for bevbert_ce/pretrain/pretrain_src/model
(pretrain_cmt.py + vilmodel.py of the continuous-environment tree).

Same class names, constructor argument, forward signatures and state_dict keys as that reference.  It differs from the
discrete model (model/pretrain_cmt.py, model/vilmodel.py) in four places, and only those are restated here:
  * the view embedding adds a LayerNorm'd depth term, LN(dep_linear(traj_view_dep_fts)), to the image term; the
    location input has angle_feat_size (4) columns and the nav-type table 2 rows (CE vilmodel.py:465-545);
  * the BEV is 11 x 11 cells at 1 m (BEV_DIM / BEV_RES), pooled without semantic labels (CE pretrain_cmt.py:100-137);
  * `GlocalTextPathCMT.forward` takes `traj_view_dep_fts` after `traj_view_img_fts` and returns (gmap_embeds,
    bev_embeds); `bev_dim` is fixed at 11 (CE vilmodel.py:715, 727-774);
  * the pre-training tasks are mlm and sap; `sap_fuse_linear` is always built (CE pretrain_cmt.py:61-86).
The CE reference's mrc, og and valid_sap_og branches call its encoder with arguments the encoder does not take
(`vp_pos_fts`, no depth features), so they cannot run there; here they raise ValueError.  Requires CUDA tensors.
"""
from collections import defaultdict

import torch
from torch import nn

from .. import blocks as Bk
from . import pretrain_cmt as discrete
from . import vilmodel
from .ops import gen_seq_masks
from .vilmodel import BertLayerNorm, BertOnlyMLMHead, PreTrainedBase, _wb

BEV_DIM = 11
BEV_RES = 1

_UNRUNNABLE = ("mrc", "og", "valid_sap_og")


class ImageEmbeddings(vilmodel.ImageEmbeddings):  # CE vilmodel.py:465-545
    def __init__(self, config):
        # Built here rather than by the discrete constructor, in the CE reference's registration order
        # (vilmodel.py:466-497): named_parameters() order is part of the drop-in contract, because the reference's
        # build_optimizer groups parameters by position and optimizer.load_state_dict restores state by position.
        nn.Module.__init__(self)
        h = config.hidden_size
        self.img_linear = nn.Linear(config.image_feat_size, h)
        self.img_layer_norm = BertLayerNorm(h, eps=1e-12)
        self.loc_linear = nn.Linear(config.angle_feat_size, h)
        self.loc_layer_norm = BertLayerNorm(h, eps=1e-12)
        if config.depth_feat_size > 0:
            self.dep_linear = nn.Linear(config.depth_feat_size, h)
            self.dep_layer_norm = BertLayerNorm(h, eps=1e-12)
        else:
            self.dep_linear = self.dep_layer_norm = None
        if config.obj_feat_size > 0 and config.obj_feat_size != config.image_feat_size:
            self.obj_linear = nn.Linear(config.obj_feat_size, h)
            self.obj_layer_norm = BertLayerNorm(h, eps=1e-12)
        else:
            self.obj_linear = self.obj_layer_norm = None
        self.nav_type_embedding = nn.Embedding(2, h)          # 0: non-navigable, 1: navigable
        self.layer_norm = BertLayerNorm(h, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.pano_encoder = vilmodel.TransformerEncoder(config, config.num_pano_layers) \
            if config.num_pano_layers > 0 else None

    def forward(self, rt, traj_view_img_fts, traj_view_dep_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, type_embed_layer):
        """-> (traj_embeds (sumP, V, H), traj_vp_lens (sumP,)), as the discrete ImageEmbeddings.  The image, depth and
        location terms, the nav-type row and the type vector are summed by one bb_add_rows3 launch."""
        if self.dep_linear is None:
            return super().forward(rt, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                                   traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, type_embed_layer)
        if traj_obj_img_fts is not None:
            raise NotImplementedError("object tokens together with depth features: the VLN-CE data has no objects "
                                      "(obj_feat_size 0)")
        lin_ln = lambda x, lin, ln, p_in=0.0: Bk.run_block(Bk.LinearLNImpl(rt, 1e-12, p_in), [x], _wb(lin) + _wb(ln))
        view = lin_ln(traj_view_img_fts, self.img_linear, self.img_layer_norm, rt.feat_p)   # drop_feats, :88-92
        dep = lin_ln(traj_view_dep_fts, self.dep_linear, self.dep_layer_norm)
        loc = lin_ln(traj_loc_fts, self.loc_linear, self.loc_layer_norm)
        emb = Bk.run_block(Bk.AddRows3Impl(vec_row=1), [view, dep, loc, traj_nav_types],
                           [self.nav_type_embedding.weight, type_embed_layer.weight])
        emb = Bk.run_block(Bk.LayerNormImpl(rt, 1e-12, self.dropout.p), [emb, None], _wb(self.layer_norm))
        if self.pano_encoder is not None:
            emb = self.pano_encoder(rt, emb, gen_seq_masks(traj_vp_view_lens, emb.shape[1]))
        return emb, traj_vp_view_lens


class GlocalTextPathCMT(vilmodel.GlocalTextPathCMT):  # CE vilmodel.py:703-841
    def __init__(self, config):
        super().__init__(config)
        self.bev_dim = 11
        self.img_embeddings = ImageEmbeddings(config)
        self.init_weights()

    def _front(self, rt, txt_ids, txt_lens, view_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types, traj_step_lens,
               traj_vp_view_lens, traj_vp_obj_lens):
        """`view_fts`: the (image, depth) feature pair, which the discrete forward / forward_mlm pass through to here
        untouched."""
        img, dep = view_fts
        txt_masks = gen_seq_masks(txt_lens, txt_ids.shape[1])
        txt = self.lang_encoder(rt, self.embeddings(rt, txt_ids), txt_masks)
        traj, traj_lens = self.img_embeddings(rt, img, dep, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                                              traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens,
                                              self.embeddings.token_type_embeddings)
        return txt, txt_masks, traj, traj_lens

    def forward(self, txt_ids, txt_lens, traj_view_img_fts, traj_view_dep_fts, traj_obj_img_fts, traj_loc_fts,
                traj_nav_types, traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids,
                gmap_lens, gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks,
                bev_nav_masks, return_gmap_embeds=True):
        gmap_embeds, bev_embeds, _, _ = super().forward(
            txt_ids, txt_lens, (traj_view_img_fts, traj_view_dep_fts), traj_obj_img_fts, traj_loc_fts, traj_nav_types,
            traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens, gmap_step_ids,
            gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks,
            return_gmap_embeds=return_gmap_embeds)
        return gmap_embeds, bev_embeds

    def forward_mlm(self, txt_ids, txt_lens, traj_view_img_fts, traj_view_dep_fts, traj_obj_img_fts, traj_loc_fts,
                    traj_nav_types, traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids,
                    gmap_lens, gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts,
                    bev_masks, bev_nav_masks):
        return super().forward_mlm(
            txt_ids, txt_lens, (traj_view_img_fts, traj_view_dep_fts), traj_obj_img_fts, traj_loc_fts, traj_nav_types,
            traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens, gmap_step_ids,
            gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks)

    def forward_sem(self, *args, **kwargs):
        raise ValueError("the VLN-CE model has no semantic-map prediction (forward_sem)")


class GlocalTextPathCMTPreTraining(discrete.GlocalTextPathCMTPreTraining):  # CE pretrain_cmt.py:61-366
    def __init__(self, config):
        PreTrainedBase.__init__(self, config)       # the discrete constructor would build the discrete encoder
        self.bert = GlocalTextPathCMT(config)
        self.bert._rt_external = True
        self.rt = self.bert.rt
        self.drop_env = nn.Dropout(config.feat_dropout)
        h = config.hidden_size
        tasks = config.pretrain_tasks
        if "mlm" in tasks:
            self.mlm_head = BertOnlyMLMHead(config)
        if "mrc" in tasks:       # parameter containers only, so that checkpoints keep the reference's keys
            self.image_classifier = discrete.RegionClassification(h, config.image_prob_size)
            if config.obj_prob_size > 0 and config.obj_prob_size != config.image_prob_size:
                self.obj_classifier = discrete.RegionClassification(h, config.obj_prob_size)
            else:
                self.obj_classifier = None
        if "sap" in tasks:
            self.global_sap_head = discrete.ClsPrediction(h)
            self.local_sap_head = discrete.ClsPrediction(h)
            self.sap_fuse_linear = discrete.ClsPrediction(h, input_size=h * 2)
        if "og" in tasks:
            self.og_head = discrete.ClsPrediction(h)
        self.init_weights()
        self.tie_weights()
        self.bev_res = BEV_RES
        self.projector, self.bev_pos_fts = discrete.build_projector(BEV_DIM, BEV_RES)

    @torch.no_grad()
    def lift_splat(self, batch):
        """CE pretrain_cmt.py:100-137 on the fused kernels: cell index straight from depth + poses, then the
        deterministic scatter-mean of the patch features; no semantic labels."""
        rgbs, depths = batch.pop("rgbs"), batch.pop("depths")
        T_c2w, T_w2c, S_w2c = batch.pop("T_c2w"), batch.pop("T_w2c"), batch.pop("S_w2c")
        gpos = batch.pop("bev_gpos_fts")
        bs = rgbs.shape[0]
        D = BEV_DIM
        idx, _ = self.projector.lift_index(depths, T_c2w, S_w2c, T_w2c, depth_scale=10.0)
        bev, _, ob, _, _ = self.projector.splat(idx, rgbs.reshape(bs, -1, rgbs.shape[-1]))
        if self.bev_pos_fts.device != bev.device:
            self.bev_pos_fts = self.bev_pos_fts.to(bev.device)
        pos = torch.cat([gpos.expand(-1, D * D, -1), self.bev_pos_fts.expand(bs, -1, -1)], dim=-1)
        batch.update({"bev_fts": bev, "bev_masks": torch.ones(bs, D * D, dtype=torch.bool, device=bev.device),
                      "bev_pos_fts": pos, "bev_ob_masks": ob, "bev_cell_idx": idx})
        return batch

    _BERT_KEYS = ("txt_ids", "txt_lens", "traj_view_img_fts", "traj_view_dep_fts", "traj_obj_img_fts", "traj_loc_fts",
                  "traj_nav_types", "traj_step_lens", "traj_vp_view_lens", "traj_vp_obj_lens", "traj_vpids",
                  "traj_cand_vpids", "gmap_lens", "gmap_step_ids", "gmap_pos_fts", "gmap_pair_dists", "gmap_vpids",
                  "bev_fts", "bev_pos_fts", "bev_masks", "bev_nav_masks")

    def forward(self, batch, task, compute_loss=True):
        if task.startswith(_UNRUNNABLE):
            self._unrunnable(task)
        if not task.startswith(("mlm", "sap")):
            raise ValueError("invalid task %r" % (task,))
        batch = defaultdict(lambda: None, batch)   # a copy: the caller's dict is left untouched, as in the reference
        self.rt.begin(self.training, tag=task)
        batch = self.lift_splat(batch)
        batch = self.drop_feats(batch)
        args = [batch[k] for k in self._BERT_KEYS]
        if task.startswith("mlm"):
            return self.forward_mlm(*args, batch["txt_labels"], compute_loss)
        return self.forward_sap(*args[:17], batch["gmap_visited_masks"], *args[17:], batch["bev_cand_idxs"],
                                batch["global_act_labels"], batch["local_act_labels"], compute_loss)

    def forward_mlm(self, txt_ids, txt_lens, traj_view_img_fts, traj_view_dep_fts, traj_obj_img_fts, traj_loc_fts,
                    traj_nav_types, traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids,
                    gmap_lens, gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts,
                    bev_masks, bev_nav_masks, txt_labels, compute_loss):
        txt_embeds = self.bert.forward_mlm(
            txt_ids, txt_lens, traj_view_img_fts, traj_view_dep_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
            traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens, gmap_step_ids,
            gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks)
        return self._mlm_head(txt_embeds, gmap_vpids, txt_labels, compute_loss)

    def forward_sap(self, txt_ids, txt_lens, traj_view_img_fts, traj_view_dep_fts, traj_obj_img_fts, traj_loc_fts,
                    traj_nav_types, traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids,
                    gmap_lens, gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, gmap_visited_masks, bev_fts,
                    bev_pos_fts, bev_masks, bev_nav_masks, bev_cand_idxs, global_act_labels, local_act_labels,
                    compute_loss):
        gmap_embeds, bev_embeds = self.bert(
            txt_ids, txt_lens, traj_view_img_fts, traj_view_dep_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
            traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens, gmap_step_ids,
            gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks)
        return self._sap_head(gmap_embeds, bev_embeds, traj_cand_vpids, gmap_lens, gmap_vpids, gmap_visited_masks,
                              bev_nav_masks, bev_cand_idxs, global_act_labels, local_act_labels, compute_loss)

    @staticmethod
    def _unrunnable(task):
        raise ValueError("task %r is not supported by the VLN-CE model: the reference's branch for it calls the encoder "
                         "with arguments its forward does not take (vp_pos_fts, no depth features)" % (task,))

    def forward_mrc(self, *args, **kwargs):
        self._unrunnable("mrc")

    def forward_og(self, *args, **kwargs):
        self._unrunnable("og")

    def forward_sap_og(self, *args, **kwargs):
        self._unrunnable("valid_sap_og")

    def forward_sem(self, *args, **kwargs):
        raise ValueError("invalid task 'sem': the VLN-CE model has no semantic-map tasks")

    forward_masksem = forward_sem
