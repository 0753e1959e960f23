"""TEST INFRASTRUCTURE ONLY -- CPU/fp32-fp64 oracle for the VLN-CE navigation network (model/ce_nav.py).

A functional restatement of bevbert_ce/vlnce_baselines/models/bev/vilmodel_cmt.py::GlocalTextPathNavCMT (line numbers
below refer to that file) over a flat ``state_dict`` with the CE network's keys, with the same three methods the CE
policy calls.  The language and cross-modal encoders, the global-map and BEV inputs, the heads and the SAP fusion are
the discrete agents' (oracle/bevbert_ref.py, `nav_forward`); the view embedding with its depth term is the CE
pre-training one (oracle/ce_ref.py), which is the same arithmetic as forward_panorama.  Pinned against the unmodified
CE reference by tests/golden/small_ce_nav.pt (tests/golden/make_ce_nav_golden.py).  The product never imports it.
"""
from oracle import bevbert_ref as R
from oracle import ce_ref as CR


class GlocalTextPathNavCMT:
    """`sd`: the network's state_dict (top-level keys, as the module's); float tensors in the oracle's dtype."""

    def __init__(self, sd, cfg):
        self.raw, self.sd, self.cfg = sd, R._nav_sd(sd), cfg

    def forward_txt(self, txt_ids, txt_masks):  # :723-727
        return R.language_encoder(self.sd, R.text_embeddings(self.sd, txt_ids, self.cfg), txt_masks, self.cfg)

    def forward_panorama(self, rgb_fts, dep_fts, loc_fts, nav_types, view_lens):  # :729-758
        b = {"traj_view_img_fts": rgb_fts, "traj_view_dep_fts": dep_fts, "traj_loc_fts": loc_fts,
             "traj_nav_types": nav_types, "traj_vp_view_lens": view_lens, "traj_step_lens": [rgb_fts.shape[0]]}
        (emb,), (lens,) = CR.image_embeddings(self.sd, b, self.cfg)
        return emb, R.seq_mask(lens)                                                         # :752-753

    def forward_navigation(self, txt_embeds, txt_masks, gmap_vpids, gmap_step_ids, gmap_img_fts, gmap_pos_fts,
                           gmap_masks, gmap_visited_masks, gmap_pair_dists, bev_fts, bev_pos_fts, bev_masks,
                           bev_nav_masks, bev_cand_idxs, bev_cand_vpids):  # :767-840
        b = {"txt_embeds": txt_embeds, "txt_masks": txt_masks, "gmap_img_embeds": gmap_img_fts,
             "gmap_step_ids": gmap_step_ids, "gmap_pos_fts": gmap_pos_fts, "gmap_masks": gmap_masks,
             "gmap_pair_dists": gmap_pair_dists, "gmap_visited_masks": gmap_visited_masks, "gmap_vpids": gmap_vpids,
             "bev_fts": bev_fts, "bev_pos_fts": bev_pos_fts, "bev_masks": bev_masks, "bev_nav_masks": bev_nav_masks,
             "bev_cand_idxs": bev_cand_idxs, "bev_cand_vpids": bev_cand_vpids, "obj_embeds": None, "obj_masks": None}
        out = R.nav_forward(self.raw, "navigation", b, self.cfg)    # the same branches, fuse and fusion rule
        del out["obj_logits"]                                         # :834-840 returns no object logits
        return out


OracleConfig = R.OracleConfig
