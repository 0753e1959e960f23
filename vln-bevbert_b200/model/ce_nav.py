"""The VLN-CE navigation network on the H100 kernels -- drop-in for
bevbert_ce/vlnce_baselines/models/bev/vilmodel_cmt.py::GlocalTextPathNavCMT, the network the R2R-CE / RxR-CE policy
(`Policy_ViewSelection_BEV`) fine-tunes and evaluates.

Same class name, constructor argument (the config of `vlnbert_init.get_vlnbert_models`), state_dict keys, shapes and
parameter order as that reference, and the three methods the policy calls:
  * `forward_txt(txt_ids, txt_masks)`                                         (vilmodel_cmt.py:723-727)
  * `forward_panorama(rgb_fts, dep_fts, loc_fts, nav_types, view_lens)`      (:729-758)
  * `forward_navigation(txt_embeds, txt_masks, gmap_vpids, gmap_step_ids, gmap_img_fts, gmap_pos_fts, gmap_masks,
    gmap_visited_masks, gmap_pair_dists, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks, bev_cand_idxs,
    bev_cand_vpids)`                                                          (:767-840)
It differs from the discrete agents' network (model/nav_vilmodel.py) in the view embedding (RGB plus an optional
LayerNorm'd depth term, switched by `use_depth_embedding`; 4 angle columns; a 2-row nav-type table; no object tokens),
in its registration order (local before global SAP head; `sap_fuse_linear` always built), in `bev_dim` fixed at 11
and in having no `fix_local_branch` / `og_head`.  The navigation step reuses the discrete body without object tokens:
the SAP fusion rule of :815-832 is the discrete one.

The policy trains these calls inside `torch.cuda.amp.autocast()` (ss_trainer_BEV.py:657); every method here runs with
autocast disabled, so outputs and gradients are the same bits with autocast on or off.  Requires CUDA tensors.
"""
import torch
from torch import nn

from .. import blocks as Bk
from . import ce_pretrain, nav_vilmodel, vilmodel
from .ops import gen_seq_masks
from .pretrain_cmt import ClsPrediction
from .vilmodel import BertLayerNorm

BEV_DIM = 11


def _no_autocast():
    return torch.autocast("cuda", enabled=False)


class ImageEmbeddings(ce_pretrain.ImageEmbeddings):  # vilmodel_cmt.py:455-486
    def __init__(self, config):
        # The CE navigation registration order (named_parameters() order is part of the drop-in contract: the
        # trainer's AdamW restores its state by position).  Depth is switched by use_depth_embedding, not by
        # depth_feat_size as in pre-training; there is no object branch.
        nn.Module.__init__(self)
        h = config.hidden_size
        self.img_linear = nn.Linear(config.image_feat_size, h)
        self.img_layer_norm = BertLayerNorm(h, eps=1e-12)
        self.loc_linear = nn.Linear(config.angle_feat_size, h)
        self.loc_layer_norm = BertLayerNorm(h, eps=1e-12)
        if config.use_depth_embedding:
            self.dep_linear = nn.Linear(config.depth_feat_size, h)
            self.dep_layer_norm = BertLayerNorm(h, eps=1e-12)
        else:
            self.dep_linear = self.dep_layer_norm = None
        self.obj_linear = self.obj_layer_norm = None
        self.nav_type_embedding = nn.Embedding(2, h)          # 0: non-navigable, 1: navigable
        self.layer_norm = BertLayerNorm(h, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.pano_encoder = vilmodel.TransformerEncoder(config, config.num_pano_layers) \
            if config.num_pano_layers > 0 else None


class GlocalTextPathNavCMT(nav_vilmodel.GlocalTextPathNavCMT):  # vilmodel_cmt.py:696-840
    def __init__(self, config):
        vilmodel.PreTrainedBase.__init__(self, config)
        h = config.hidden_size
        self.bev_dim = BEV_DIM
        self.embeddings = vilmodel.BertEmbeddings(config)
        self.lang_encoder = vilmodel.LanguageEncoder(config)
        self.img_embeddings = ImageEmbeddings(config)
        self.local_encoder = vilmodel.LocalBEVEncoder(config)
        self.local_encoder.bev_dim = BEV_DIM
        self.global_encoder = vilmodel.GlobalMapEncoder(config)
        self.local_sap_head = ClsPrediction(h)
        self.global_sap_head = ClsPrediction(h)
        self.sap_fuse_linear = ClsPrediction(h, input_size=h * 2)
        self.rt = Bk.Runtime()
        self.init_weights()
        fix = lambda mods: [p.requires_grad_(False) for m in mods for p in m.parameters()]
        if config.fix_lang_embedding:
            fix([self.embeddings, self.lang_encoder])
        if config.fix_pano_embedding:
            fix([self.img_embeddings])

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path=None, config=None, state_dict=None, **kw):
        """Loads `state_dict` the way the reference (a transformers BertPreTrainedModel with base_model_prefix `bert`,
        which it has no child of) does: when any key starts with `bert`, only the `bert.`-prefixed keys are read, with
        the prefix removed; otherwise every key is read as it is.  Keys the network does not have are ignored, and a
        key it has with another shape raises RuntimeError.  `get_vlnbert_models` puts `bert.` before the head keys of
        a CE pre-training checkpoint (vlnbert_init.py:21-30), so its encoder and SAP heads all land."""
        model = cls(config)
        if state_dict is not None:
            if any(k.startswith("bert") for k in state_dict):
                state_dict = {k[5:]: v for k, v in state_dict.items() if k.startswith("bert.")}
            own = model.state_dict()
            bad = ["%s: checkpoint %s, network %s" % (k, tuple(v.shape), tuple(own[k].shape))
                   for k, v in state_dict.items() if k in own and v.shape != own[k].shape]
            if bad:
                raise RuntimeError("size mismatch loading %s: %s" % (cls.__name__, "; ".join(bad)))
            model.load_state_dict({k: v for k, v in state_dict.items() if k in own}, strict=False)
        return model

    # ------------------------------------------------------------------------------------------ the policy's calls
    def forward_txt(self, txt_ids, txt_masks):
        with _no_autocast():
            return self.forward_text(txt_ids, txt_masks)

    def forward_panorama(self, rgb_fts, dep_fts, loc_fts, nav_types, view_lens, vtot=None):
        """-> (pano_embeds fp32 (B, V, H), pano_masks bool (B, W)).  W is max(view_lens) as in the reference, read from
        the device; a caller that knows it (the padded width of its inputs) passes it as `vtot`, which keeps the call
        free of host synchronisations (CUDA-graph capture)."""
        with _no_autocast():
            rt = self.rt
            rt.begin(self.training)
            rt.feat_p = 0.0          # the policy applies no feature dropout inside the network
            emb, lens = self.img_embeddings(rt, rgb_fts, dep_fts, None, loc_fts, nav_types, None, view_lens, None,
                                            self.embeddings.token_type_embeddings)
            width = int(view_lens.max()) if vtot is None else vtot
            return Bk.to_f32(emb), gen_seq_masks(lens, width)

    def forward_navigation(self, txt_embeds, txt_masks, gmap_vpids, gmap_step_ids, gmap_img_fts, gmap_pos_fts,
                           gmap_masks, gmap_visited_masks, gmap_pair_dists, bev_fts, bev_pos_fts, bev_masks,
                           bev_nav_masks, bev_cand_idxs, bev_cand_vpids):
        """-> {gmap_embeds, global_logits, local_logits, fused_logits}, as the reference (no object logits).
        `bev_cand_idxs` may be on the host: the trainer's `_nav_bev_variable` leaves it there (ss_trainer_BEV.py:511)."""
        bev_cand_idxs = bev_cand_idxs.to(txt_embeds.device)
        with _no_autocast():
            out = self.forward_navigation_per_step(
                txt_embeds, txt_masks, gmap_img_fts, gmap_step_ids, gmap_pos_fts, gmap_masks, gmap_pair_dists,
                gmap_visited_masks, gmap_vpids, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks, bev_cand_idxs,
                bev_cand_vpids, None, None)
        del out["obj_logits"]
        return out

    def forward(self, mode, batch, **kwargs):
        raise NotImplementedError(
            "the VLN-CE navigation network is called through forward_txt, forward_panorama and forward_navigation; "
            "its reference forward(mode, batch) calls methods the class does not define (vilmodel_cmt.py:842-863)")
