"""GlocalTextPathNavCMT on the H100 kernels -- the agents' per-step API (map_nav_src/models/vilmodel.py:705-912):
`forward(mode, batch)` with mode in {'language', 'panorama', 'navigation'}.  Same parameter names as the reference
(heads live at the top level, as after `vlnbert_init.py:39-46` re-prefixing).  Tensors crossing the API are fp32
like the reference's (the agents average / cache them on the host side); inside, activations are bf16."""
import torch
from torch import nn

from .. import blocks as Bk
from .ops import build_sap_fusion, gen_seq_masks
from .pretrain_cmt import ClsPrediction
from .vilmodel import (BertEmbeddings, GlobalMapEncoder, ImageEmbeddings, LanguageEncoder, LocalBEVEncoder,
                       PreTrainedBase, _wb)


class GlocalTextPathNavCMT(PreTrainedBase):
    def __init__(self, config):
        super().__init__(config)
        self.bev_dim = config.bev_dim
        self.embeddings = BertEmbeddings(config)
        self.lang_encoder = LanguageEncoder(config)
        self.img_embeddings = ImageEmbeddings(config)
        self.local_encoder = LocalBEVEncoder(config)
        self.global_encoder = GlobalMapEncoder(config)
        h = config.hidden_size
        self.global_sap_head = ClsPrediction(h)
        self.local_sap_head = ClsPrediction(h)
        self.sap_fuse_linear = ClsPrediction(h, input_size=h * 2) if config.glocal_fuse else None
        if config.obj_feat_size > 0:
            self.og_head = ClsPrediction(h)
        self.rt = Bk.Runtime()
        self.init_weights()
        fix = lambda mods: [p.requires_grad_(False) for m in mods for p in m.parameters()]
        if getattr(config, "fix_lang_embedding", False) or getattr(config, "fix_local_branch", False):
            fix([self.embeddings, self.lang_encoder])
        if getattr(config, "fix_pano_embedding", False) or getattr(config, "fix_local_branch", False):
            fix([self.img_embeddings])
        if getattr(config, "fix_local_branch", False):
            fix([self.local_encoder, self.local_sap_head] + ([self.og_head] if hasattr(self, "og_head") else []))

    # ------------------------------------------------------------------------------------------ modes
    def forward_text(self, txt_ids, txt_masks):
        rt = self.rt
        rt.begin(self.training)
        return Bk.to_f32(self.lang_encoder(rt, self.embeddings(rt, txt_ids), txt_masks))

    def forward_panorama_per_step(self, view_img_fts, obj_img_fts, loc_fts, nav_types, view_lens, obj_lens, vtot=None):
        """`vtot`: token width with objects (see ImageEmbeddings.forward); None reads max(view + object lens)."""
        rt = self.rt
        rt.begin(self.training)
        rt.feat_p = 0.0          # the agents apply feature dropout themselves (map_nav_src/models/model.py:21-41)
        emb, lens = self.img_embeddings(rt, view_img_fts, obj_img_fts, loc_fts, nav_types, None, view_lens, obj_lens,
                                        self.embeddings.token_type_embeddings, vtot=vtot)
        return Bk.to_f32(emb), gen_seq_masks(lens, emb.shape[1])

    def forward_navigation_per_step(self, txt_embeds, txt_masks, gmap_img_embeds, gmap_step_ids, gmap_pos_fts,
                                    gmap_masks, gmap_pair_dists, gmap_visited_masks, gmap_vpids, bev_fts, bev_pos_fts,
                                    bev_masks, bev_nav_masks, bev_cand_idxs, bev_cand_vpids, obj_embeds, obj_masks):
        rt = self.rt
        rt.begin(self.training)
        rt.feat_p = 0.0
        B = txt_embeds.size(0)
        dev = txt_embeds.device
        txt = Bk.to_act(txt_embeds)
        ge = self.global_encoder
        pos = Bk.run_block(Bk.LinearLNImpl(rt, 1e-12), [gmap_pos_fts],
                           _wb(ge.gmap_pos_embeddings[0]) + _wb(ge.gmap_pos_embeddings[1]))
        g_in = Bk.run_block(Bk.AddRowsImpl(), [Bk.to_act(gmap_img_embeds), pos, gmap_step_ids],
                            [ge.gmap_step_embeddings.weight, None])
        gmap_embeds = ge.encoder(rt, txt, txt_masks, g_in, gmap_masks, graph_sprels=ge.graph_bias(gmap_pair_dists))
        obj_in = Bk.to_act(obj_embeds) if obj_embeds is not None else None
        bev_embeds, obj_out = self.local_encoder(rt, txt, txt_masks, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks,
                                                 obj_in, obj_masks)
        G, Kc = gmap_embeds.shape[1], bev_cand_idxs.shape[1]
        n = self.bev_dim * self.bev_dim
        Hd = gmap_embeds.shape[-1]
        bev_flat = bev_embeds.contiguous().view(-1, Hd)
        ar = torch.arange(B, device=dev)
        cand_embeds = Bk.run_block(Bk.GatherRowsImpl(), [bev_flat, (ar[:, None] * n + bev_cand_idxs).reshape(-1)], [])
        cand_masks = bev_nav_masks[ar[:, None], bev_cand_idxs]
        if self.sap_fuse_linear is None:
            fuse = 0.5
        else:
            g0 = Bk.run_block(Bk.GatherRowsImpl(), [gmap_embeds.reshape(-1, Hd), ar * G], [])
            c0 = Bk.run_block(Bk.GatherRowsImpl(), [bev_flat, ar * n + (n - 1) // 2], [])
            fuse = torch.sigmoid(self.sap_fuse_linear(rt, torch.cat([g0, c0], 1)))
        global_logits = self.global_sap_head(rt, gmap_embeds).squeeze(2) * fuse
        global_logits = global_logits.masked_fill(gmap_visited_masks, -float("inf"))
        global_logits = global_logits.masked_fill(gmap_masks.logical_not(), -float("inf"))
        local_logits = self.local_sap_head(rt, cand_embeds).view(B, Kc) * (1 - fuse)
        local_logits = local_logits.masked_fill(cand_masks.logical_not(), -float("inf"))
        # bev_cand_vpids[i][0] is the [stop] slot (reference loop skips j == 0)
        Fm = build_sap_fusion(gmap_vpids, gmap_visited_masks, [c[1:] for c in bev_cand_vpids], G, Kc, dev)
        fused_logits = global_logits + torch.einsum("bgk,bk->bg", Fm, local_logits.masked_fill(cand_masks.logical_not(), 0.0))
        fused_logits = torch.cat([torch.where(torch.isinf(local_logits[:, :1]), local_logits[:, :1], fused_logits[:, :1]),
                                  fused_logits[:, 1:]], 1)
        obj_logits = None
        if obj_out is not None:
            obj_logits = self.og_head(rt, obj_out.contiguous()).squeeze(2).masked_fill(obj_masks.logical_not(), -float("inf"))
        return {"gmap_embeds": Bk.to_f32(gmap_embeds), "global_logits": global_logits, "local_logits": local_logits,
                "fused_logits": fused_logits, "obj_logits": obj_logits}

    def forward(self, mode, batch, **kwargs):
        if mode == "language":
            return self.forward_text(batch["txt_ids"], batch["txt_masks"])
        if mode == "panorama":
            return self.forward_panorama_per_step(batch["view_img_fts"], batch["obj_img_fts"], batch["loc_fts"],
                                                  batch["nav_types"], batch["view_lens"], batch["obj_lens"])
        if mode == "navigation":
            return self.forward_navigation_per_step(
                batch["txt_embeds"], batch["txt_masks"], batch["gmap_img_embeds"], batch["gmap_step_ids"],
                batch["gmap_pos_fts"], batch["gmap_masks"], batch["gmap_pair_dists"], batch["gmap_visited_masks"],
                batch["gmap_vpids"], batch["bev_fts"], batch["bev_pos_fts"], batch["bev_masks"], batch["bev_nav_masks"],
                batch["bev_cand_idxs"], batch["bev_cand_vpids"], batch["obj_embeds"], batch["obj_masks"])
        raise NotImplementedError(mode)
