"""TEST INFRASTRUCTURE ONLY -- CPU/fp32 oracle for the VLN-CE pre-training model (model/ce_pretrain.py).

A functional restatement of bevbert_ce/pretrain/pretrain_src/model (paths below are relative to that directory) over a
flat ``state_dict`` with the CE reference's keys.  Everything the CE model shares with the discrete one (language,
panorama, cross-modal encoders, global-map input, BEV input, heads, SAP fusion, lifting geometry) is taken from
oracle/bevbert_ref.py; this file restates only what differs: the depth term of the view embedding, the semantics-free
lift-splat at 11 x 11 / 1 m, and the task dispatch.  Pinned against the unmodified CE reference by
tests/golden/small_ce.pt (tests/golden/make_ce_golden.py).  The product package never imports it.
"""
import torch
import torch.nn.functional as F

from oracle import bevbert_ref as R

BEV_DIM = 11    # pretrain_cmt.py:16-17
BEV_RES = 1


def image_embeddings(sd, b, cfg):  # ImageEmbeddings.forward, vilmodel.py:499-545 (no object tokens)
    p = "bert.img_embeddings"
    if b.get("traj_obj_img_fts") is not None:
        raise NotImplementedError("object tokens: the VLN-CE data has none")
    view = R._ln(sd, p + ".img_layer_norm", R._lin(sd, p + ".img_linear", b["traj_view_img_fts"]), 1e-12)
    if (p + ".dep_linear.weight") in sd:                                                     # :507-509
        view = view + R._ln(sd, p + ".dep_layer_norm", R._lin(sd, p + ".dep_linear", b["traj_view_dep_fts"]), 1e-12)
    lens = b["traj_vp_view_lens"]
    emb = view + R._ln(sd, p + ".loc_layer_norm", R._lin(sd, p + ".loc_linear", b["traj_loc_fts"]), 1e-12) + \
        sd[p + ".nav_type_embedding.weight"][b["traj_nav_types"]] + \
        sd["bert.embeddings.token_type_embeddings.weight"][1][None, None]                     # :530-533
    emb = R._drop(R._ln(sd, p + ".layer_norm", emb, 1e-12), cfg.drop_p)
    masks = R.seq_mask(lens)
    if cfg.num_pano_layers > 0:
        for i in range(cfg.num_pano_layers):
            emb = R.pano_layer(sd, "%s.pano_encoder.layers.%d" % (p, i), emb, ~masks, cfg)
        emb = R._ln(sd, p + ".pano_encoder.norm", emb, 1e-12)
    steps = list(b["traj_step_lens"])
    return torch.split(emb, steps, 0), torch.split(lens, steps, 0)


def lift_splat(b):
    """pretrain_cmt.py:100-137: the discrete lifting geometry at BEV_DIM / BEV_RES, features only."""
    rgbs, depths = b.pop("rgbs"), b.pop("depths")
    T_c2w, T_w2c, S_w2c, gpos = b.pop("T_c2w"), b.pop("T_w2c"), b.pop("S_w2c"), b.pop("bev_gpos_fts")
    B, D = rgbs.shape[0], BEV_DIM
    pc, nod = R.lift_points(depths, T_c2w, S_w2c, T_w2c)
    idx = R.cell_index(pc, nod, D, BEV_RES)
    feat = rgbs.reshape(B, -1, rgbs.shape[-1])
    bev = torch.stack([R.scatter_mean(feat[i], idx[i], D * D) for i in range(B)], 0)
    b["bev_cell_idx"] = idx
    b["bev_fts"] = bev
    b["bev_masks"] = torch.ones(B, D * D, dtype=torch.bool)                                      # :126
    b["bev_pos_fts"] = torch.cat([gpos.expand(-1, D * D, -1),
                                  R.bevpos_polar(D).reshape(1, D * D, 3).expand(B, -1, -1)], -1)   # :129-130
    return b


def _front(sd, b, cfg):
    txt_masks = R.seq_mask(b["txt_lens"])
    txt = R.language_encoder(sd, R.text_embeddings(sd, b["txt_ids"], cfg), txt_masks, cfg)
    split_embeds, split_lens = image_embeddings(sd, b, cfg)
    return txt, txt_masks, split_embeds, split_lens


def encode(sd, b, cfg):  # GlocalTextPathCMT.forward, vilmodel.py:726-774 -> (gmap_embeds, bev_embeds)
    txt, txt_masks, se, sl = _front(sd, b, cfg)
    g, gm = R.gmap_input(sd, se, sl, b)
    gmap = R.crossmodal_encoder(sd, "bert.global_encoder.encoder", txt, txt_masks, g, gm, R.graph_sprels(sd, b), cfg)
    bev, _ = R._local(sd, b, txt, txt_masks, None, None, cfg)
    return gmap, bev


def encode_mlm(sd, b, cfg):  # GlocalTextPathCMT.forward_mlm, vilmodel.py:777-839
    txt, txt_masks, se, sl = _front(sd, b, cfg)
    tm = R.neg_mask(txt_masks)
    g, gm = R.gmap_input(sd, se, sl, b)
    gmn = R.neg_mask(gm)
    gt = txt
    for i in range(cfg.num_x_layers):
        gt = R.xlayer_lang2visn(sd, "bert.global_encoder.encoder.x_layers.%d" % i, gt, tm, g, gmn, cfg)
    bev, bm = R.bev_input(sd, b), R.neg_mask(b["bev_masks"])
    bt = txt
    for i in range(cfg.num_x_layers):
        bt = R.xlayer_lang2visn(sd, "bert.local_encoder.encoder.x_layers.%d" % i, bt, tm, bev, bm, cfg)
    return gt + bt


def forward(sd, batch, task, cfg, compute_loss=True):
    """GlocalTextPathCMTPreTraining.forward, pretrain_cmt.py:139-201 (+ forward_mlm :203-227, forward_sap :294-366).
    mrc, og and valid_sap_og raise ValueError: their reference branches cannot run (see model/ce_pretrain.py)."""
    if task.startswith(("mrc", "og", "valid_sap_og")):
        raise ValueError("task %r cannot run in the VLN-CE reference" % (task,))
    if not task.startswith(("mlm", "sap")):
        raise ValueError("invalid task")
    b = lift_splat(dict(batch))
    if cfg.feat_drop_p > 0:  # drop_feats, :88-92
        for k in ("traj_view_img_fts", "bev_fts"):
            b[k] = R._drop(b[k], cfg.feat_drop_p)
    if task.startswith("mlm"):
        txt = encode_mlm(sd, b, cfg)
        sel = b["txt_labels"] != -1
        scores = R.mlm_head(sd, txt[sel], cfg)
        return F.cross_entropy(scores, b["txt_labels"][sel], reduction="none") if compute_loss else scores
    gmap, bev = encode(sd, b, cfg)
    gl, ll, fl = R.sap_logits(sd, b, cfg, gmap, bev)
    if not compute_loss:
        return gl, ll, fl, b["global_act_labels"], b["local_act_labels"]
    return F.cross_entropy(gl, b["global_act_labels"], reduction="none") + \
        F.cross_entropy(ll, b["local_act_labels"], reduction="none") + \
        F.cross_entropy(fl, b["global_act_labels"], reduction="none")


OracleConfig = R.OracleConfig
