"""GlocalTextPathCMT on the H100 kernels -- drop-in for pretrain_src/model/vilmodel.py.

Same class names, constructor argument (an HF-style config), forward signatures and state_dict keys as the
reference (SURVEY.md 8b); the nn.Linear / nn.LayerNorm / nn.Embedding / nn.MultiheadAttention children are
parameter containers only -- all arithmetic runs in the sm_90a kernels through `blocks.run_block`.
nn.Dropout children are kept so that the reference's `set_dropout(model, p)` (utils/misc.py:19-25) still
controls the probabilities.
"""
import torch
from torch import nn

from .. import blocks as Bk
from .ops import build_gmap_segments, finish_gmap_segments, gen_seq_masks, inf_key_mask, neg_key_mask

BertLayerNorm = nn.LayerNorm


def _wb(m):
    return [m.weight, m.bias]


# ------------------------------------------------------------------------------------------------ containers
class BertEmbeddings(nn.Module):  # vilmodel.py:48-77
    def __init__(self, config):
        super().__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size, padding_idx=0)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=config.layer_norm_eps)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.eps = config.layer_norm_eps

    def forward(self, rt, input_ids):
        impl = Bk.TextEmbedImpl(rt, self.eps, self.dropout.p)
        return Bk.run_block(impl, [input_ids], [self.word_embeddings.weight, self.position_embeddings.weight,
                                                self.token_type_embeddings.weight] + _wb(self.LayerNorm))


class BertSelfAttention(nn.Module):  # :79-141
    def __init__(self, config):
        super().__init__()
        self.num_attention_heads = config.num_attention_heads
        self.query = nn.Linear(config.hidden_size, config.hidden_size)
        self.key = nn.Linear(config.hidden_size, config.hidden_size)
        self.value = nn.Linear(config.hidden_size, config.hidden_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)

    def params(self):
        return _wb(self.query) + _wb(self.key) + _wb(self.value)


class BertSelfOutput(nn.Module):  # :143-154
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=config.layer_norm_eps)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def params(self):
        return _wb(self.dense) + _wb(self.LayerNorm)


class BertAttention(nn.Module):  # :156-166
    def __init__(self, config):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)

    def params(self):
        return self.self.params() + self.output.params()


class BertIntermediate(nn.Module):  # :168-180
    def __init__(self, config):
        super().__init__()
        if config.hidden_act not in ("gelu",):
            raise NotImplementedError("the fused FFN kernel implements the exact-erf GELU of the shipped configs")
        self.dense = nn.Linear(config.hidden_size, config.intermediate_size)


class BertOutput(nn.Module):  # :182-193
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.intermediate_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=config.layer_norm_eps)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


def _run_bert_layer(rt, eps, heads, att, inter, out, x, kmask, bias=None):
    impl = Bk.BertLayerImpl(rt, heads, eps, att.self.dropout.p, att.output.dropout.p)
    params = att.params() + _wb(inter.dense) + _wb(out.dense) + _wb(out.LayerNorm)
    return Bk.run_block(impl, [x, kmask, bias], params)


class BertLayer(nn.Module):  # :195-208
    def __init__(self, config):
        super().__init__()
        self.attention = BertAttention(config)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)
        self.eps, self.heads = config.layer_norm_eps, config.num_attention_heads

    def forward(self, rt, hidden_states, key_mask):
        return _run_bert_layer(rt, self.eps, self.heads, self.attention, self.intermediate, self.output, hidden_states,
                               key_mask)


class BertPredictionHeadTransform(nn.Module):  # :258-272
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=config.layer_norm_eps)


class BertLMPredictionHead(nn.Module):  # :274-290
    def __init__(self, config):
        super().__init__()
        self.transform = BertPredictionHeadTransform(config)
        self.decoder = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.bias = nn.Parameter(torch.zeros(config.vocab_size))


class BertOnlyMLMHead(nn.Module):  # :292-299
    def __init__(self, config):
        super().__init__()
        self.predictions = BertLMPredictionHead(config)
        self.eps = config.layer_norm_eps

    def params(self):
        pr = self.predictions
        return _wb(pr.transform.dense) + _wb(pr.transform.LayerNorm) + [pr.decoder.weight, pr.bias]


class BertOutAttention(nn.Module):  # :301-352
    def __init__(self, config, ctx_dim=None):
        super().__init__()
        ctx_dim = config.hidden_size if ctx_dim is None else ctx_dim
        self.query = nn.Linear(config.hidden_size, config.hidden_size)
        self.key = nn.Linear(ctx_dim, config.hidden_size)
        self.value = nn.Linear(ctx_dim, config.hidden_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)


class BertXAttention(nn.Module):  # :354-363
    def __init__(self, config, ctx_dim=None):
        super().__init__()
        self.att = BertOutAttention(config, ctx_dim=ctx_dim)
        self.output = BertSelfOutput(config)
        self.eps, self.heads = config.layer_norm_eps, config.num_attention_heads

    def forward(self, rt, input_tensor, ctx_tensor, ctx_key_mask=None):
        impl = Bk.XAttnImpl(rt, self.heads, self.eps, self.att.dropout.p, self.output.dropout.p)
        params = _wb(self.att.query) + _wb(self.att.key) + _wb(self.att.value) + self.output.params()
        return Bk.run_block(impl, [input_tensor, ctx_tensor, ctx_key_mask], params)


class GraphLXRTXLayer(nn.Module):  # :365-421
    def __init__(self, config):
        super().__init__()
        if config.use_lang2visn_attn:
            self.lang_self_att = BertAttention(config)
            self.lang_inter = BertIntermediate(config)
            self.lang_output = BertOutput(config)
        self.visn_self_att = BertAttention(config)
        self.visn_inter = BertIntermediate(config)
        self.visn_output = BertOutput(config)
        self.visual_attention = BertXAttention(config)
        self.eps, self.heads = config.layer_norm_eps, config.num_attention_heads

    def forward(self, rt, lang_feats, lang_key_mask, visn_feats, visn_key_mask, graph_sprels=None):
        v = self.visual_attention(rt, visn_feats, lang_feats, lang_key_mask)
        return _run_bert_layer(rt, self.eps, self.heads, self.visn_self_att, self.visn_inter, self.visn_output, v,
                               visn_key_mask, graph_sprels)

    def forward_lang2visn(self, rt, lang_feats, lang_key_mask, visn_feats, visn_key_mask):
        l = self.visual_attention(rt, lang_feats, visn_feats, visn_key_mask)
        return _run_bert_layer(rt, self.eps, self.heads, self.lang_self_att, self.lang_inter, self.lang_output, l,
                               lang_key_mask)

    def forward_visn2visn(self, rt, visn_feats, visn_key_mask):
        return _run_bert_layer(rt, self.eps, self.heads, self.visn_self_att, self.visn_inter, self.visn_output,
                               visn_feats, visn_key_mask)


class LanguageEncoder(nn.Module):  # :424-444
    def __init__(self, config):
        super().__init__()
        self.num_l_layers = config.num_l_layers
        self.update_lang_bert = config.update_lang_bert
        self.layer = nn.ModuleList([BertLayer(config) for _ in range(self.num_l_layers)])
        if not self.update_lang_bert:
            for p in self.layer.parameters():
                p.requires_grad = False

    def forward(self, rt, txt_embeds, txt_masks):
        km = neg_key_mask(txt_masks)
        for layer in self.layer:
            txt_embeds = layer(rt, txt_embeds, km)
        return txt_embeds if self.update_lang_bert else txt_embeds.detach()


class CrossmodalEncoder(nn.Module):  # :446-463
    def __init__(self, config):
        super().__init__()
        self.num_x_layers = config.num_x_layers
        self.x_layers = nn.ModuleList([GraphLXRTXLayer(config) for _ in range(self.num_x_layers)])

    def forward(self, rt, txt_embeds, txt_masks, img_embeds, img_masks, graph_sprels=None):
        tk, ik = neg_key_mask(txt_masks), neg_key_mask(img_masks)
        for layer in self.x_layers:
            img_embeds = layer(rt, txt_embeds, tk, img_embeds, ik, graph_sprels=graph_sprels)
        return img_embeds


# ------------------------------------------------------------------------------------------------ panorama encoder
class TransformerEncoderLayer(nn.Module):  # transformer.py:133-190 (pre-norm variant only)
    def __init__(self, d_model, nhead, dim_feedforward, dropout):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)
        self.dropout1 = nn.Dropout(dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.nhead = nhead

    def params(self):
        a = self.self_attn
        return [a.in_proj_weight, a.in_proj_bias, a.out_proj.weight, a.out_proj.bias] + _wb(self.linear1) + \
            _wb(self.linear2) + _wb(self.norm1) + _wb(self.norm2)

    def forward(self, rt, x, key_mask):
        impl = Bk.PanoLayerImpl(rt, self.nhead, self.self_attn.dropout, self.dropout.p)
        return Bk.run_block(impl, [x, key_mask], self.params())


class TransformerEncoder(nn.Module):  # transformer.py:62-89, ops.py:11-23
    def __init__(self, config, num_layers):
        super().__init__()
        self.layers = nn.ModuleList([TransformerEncoderLayer(config.hidden_size, config.num_attention_heads,
                                                             config.intermediate_size, config.hidden_dropout_prob)
                                     for _ in range(num_layers)])
        self.norm = BertLayerNorm(config.hidden_size, eps=1e-12)

    def forward(self, rt, x, valid_masks):
        km = inf_key_mask(valid_masks)
        for layer in self.layers:
            x = layer(rt, x, km)
        return Bk.run_block(Bk.LayerNormImpl(rt, 1e-12), [x, None], _wb(self.norm))


class ImageEmbeddings(nn.Module):  # vilmodel.py:465-536
    def __init__(self, config):
        super().__init__()
        self.img_linear = nn.Linear(config.image_feat_size, config.hidden_size)
        self.img_layer_norm = BertLayerNorm(config.hidden_size, eps=1e-12)
        self.loc_linear = nn.Linear(config.angle_feat_size + 3, config.hidden_size)
        self.loc_layer_norm = BertLayerNorm(config.hidden_size, eps=1e-12)
        if config.obj_feat_size > 0 and config.obj_feat_size != config.image_feat_size:
            self.obj_linear = nn.Linear(config.obj_feat_size, config.hidden_size)
            self.obj_layer_norm = BertLayerNorm(config.hidden_size, eps=1e-12)
        else:
            self.obj_linear = self.obj_layer_norm = None
        self.nav_type_embedding = nn.Embedding(3, config.hidden_size)
        self.layer_norm = BertLayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.pano_encoder = TransformerEncoder(config, config.num_pano_layers) if config.num_pano_layers > 0 else None

    def forward(self, rt, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types, traj_step_lens,
                traj_vp_view_lens, traj_vp_obj_lens, type_embed_layer, vtot=None):
        """-> (traj_embeds (sumP, Vtot, H) flat over panoramas, traj_vp_lens (sumP,)); the reference returns
        the same data split per sample (torch.split by traj_step_lens).  With objects, Vtot is max(view + object
        lens), read from the device; a caller that knows a width >= that (the padded width of `traj_loc_fts`) passes it
        as `vtot`, which keeps the call free of host synchronisations (CUDA-graph capture)."""
        dev = traj_view_img_fts.device
        lin_ln = lambda x, lin, ln, p_in=0.0: Bk.run_block(Bk.LinearLNImpl(rt, 1e-12, p_in), [x], _wb(lin) + _wb(ln))
        view = lin_ln(traj_view_img_fts, self.img_linear, self.img_layer_norm, rt.feat_p)
        if traj_obj_img_fts is not None:
            if self.obj_linear is None:
                obj = lin_ln(traj_obj_img_fts, self.img_linear, self.img_layer_norm, rt.feat_p)
            else:
                obj = lin_ln(traj_obj_img_fts, self.obj_linear, self.obj_layer_norm, rt.feat_p)
            nP, V, Hd = view.shape
            O = obj.shape[1]
            lens = traj_vp_view_lens + traj_vp_obj_lens
            Vtot = int(lens.max()) if vtot is None else vtot
            ar = torch.arange(Vtot, device=dev)[None, :]
            base = torch.arange(nP, device=dev)[:, None]
            vl, ol = traj_vp_view_lens[:, None], traj_vp_obj_lens[:, None]
            src = torch.where(ar < vl, base * V + ar, nP * V + base * O + (ar - vl))
            src = torch.where(ar < vl + ol, src, torch.full_like(src, -1)).reshape(-1)
            both = torch.cat([view.reshape(-1, Hd), obj.reshape(-1, Hd)], 0)
            img = Bk.run_block(Bk.GatherRowsImpl(), [both, src], []).view(nP, Vtot, Hd)
        else:
            img, lens = view, traj_vp_view_lens
        loc = lin_ln(traj_loc_fts, self.loc_linear, self.loc_layer_norm)
        emb = Bk.run_block(Bk.AddRowsImpl(vec_row=1), [img, loc, traj_nav_types],
                           [self.nav_type_embedding.weight, type_embed_layer.weight])
        emb = Bk.run_block(Bk.LayerNormImpl(rt, 1e-12, self.dropout.p), [emb, None], _wb(self.layer_norm))
        if self.pano_encoder is not None:
            emb = self.pano_encoder(rt, emb, gen_seq_masks(lens, emb.shape[1]))
        return emb, lens


class LocalBEVEncoder(nn.Module):  # :572-615
    def __init__(self, config):
        super().__init__()
        self.bev_dim = config.bev_dim
        self.bev_fts_embeddings = nn.Sequential(nn.Linear(768, config.hidden_size),
                                                BertLayerNorm(config.hidden_size, eps=1e-12))
        self.bev_pos_embeddings = nn.Sequential(nn.Linear(3 + 7, config.hidden_size),
                                                BertLayerNorm(config.hidden_size, eps=1e-12))
        self.nav_type_embedding = nn.Embedding(2, config.hidden_size)
        self.encoder = CrossmodalEncoder(config)

    def bev_input_embedding(self, rt, bev_fts, bev_pos_fts, bev_nav_masks):
        f = Bk.run_block(Bk.LinearLNImpl(rt, 1e-12, rt.feat_p), [bev_fts],
                         _wb(self.bev_fts_embeddings[0]) + _wb(self.bev_fts_embeddings[1]))
        p = Bk.run_block(Bk.LinearLNImpl(rt, 1e-12), [bev_pos_fts],
                         _wb(self.bev_pos_embeddings[0]) + _wb(self.bev_pos_embeddings[1]))
        return Bk.run_block(Bk.AddRowsImpl(), [f, p, bev_nav_masks.long()], [self.nav_type_embedding.weight, None])

    def forward(self, rt, txt_embeds, txt_masks, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks, obj_embeds, obj_masks):
        bev = self.bev_input_embedding(rt, bev_fts, bev_pos_fts, bev_nav_masks)
        if obj_embeds is not None:
            bev = torch.cat([bev, obj_embeds], dim=1)
            bev_masks = torch.cat([bev_masks, obj_masks], dim=1)
        out = self.encoder(rt, txt_embeds, txt_masks, bev, bev_masks)
        n = self.bev_dim * self.bev_dim
        return out[:, :n], (out[:, n:] if obj_embeds is not None else None)


class GlobalMapEncoder(nn.Module):  # :617-700
    def __init__(self, config):
        super().__init__()
        self.gmap_pos_embeddings = nn.Sequential(nn.Linear(config.angle_feat_size + 3, config.hidden_size),
                                                 BertLayerNorm(config.hidden_size, eps=1e-12))
        self.gmap_step_embeddings = nn.Embedding(config.max_action_steps, config.hidden_size)
        self.encoder = CrossmodalEncoder(config)
        self.sprel_linear = nn.Linear(1, 1) if config.graph_sprels else None

    def gmap_input_embedding(self, rt, traj_embeds, traj_vp_lens, traj_step_lens, traj_vpids, traj_cand_vpids,
                             gmap_vpids, gmap_step_ids, gmap_pos_fts, gmap_lens):
        B, G = gmap_step_ids.shape
        nP, Vtot, Hd = traj_embeds.shape
        pre = getattr(gmap_vpids, "host_segments", None)      # PreparedList from prepare_batch(): host work already done
        if pre is not None and pre[0] == (G, Vtot):
            seg = finish_gmap_segments(pre[1], traj_vp_lens, Vtot, traj_embeds.device)
        else:
            seg = build_gmap_segments(traj_step_lens, traj_vp_lens, traj_vpids, traj_cand_vpids, gmap_vpids, G,
                                      Vtot, traj_embeds.device)
        agg = Bk.run_block(Bk.SegmentSumImpl(), [traj_embeds.reshape(-1, Hd), *seg], []).view(B, G, Hd)
        pos = Bk.run_block(Bk.LinearLNImpl(rt, 1e-12), [gmap_pos_fts],
                           _wb(self.gmap_pos_embeddings[0]) + _wb(self.gmap_pos_embeddings[1]))
        emb = Bk.run_block(Bk.AddRowsImpl(), [agg, pos, gmap_step_ids], [self.gmap_step_embeddings.weight, None])
        return emb, gen_seq_masks(gmap_lens, G)

    def graph_bias(self, gmap_pair_dists):
        if self.sprel_linear is None:
            return None
        return (gmap_pair_dists * self.sprel_linear.weight.view(1, 1, 1) + self.sprel_linear.bias.view(1, 1, 1)).contiguous()

    def forward(self, rt, txt_embeds, txt_masks, traj_embeds, traj_vp_lens, traj_step_lens, traj_vpids,
                traj_cand_vpids, gmap_vpids, gmap_step_ids, gmap_pos_fts, gmap_lens, graph_sprels=None):
        emb, masks = self.gmap_input_embedding(rt, traj_embeds, traj_vp_lens, traj_step_lens, traj_vpids,
                                               traj_cand_vpids, gmap_vpids, gmap_step_ids, gmap_pos_fts, gmap_lens)
        return self.encoder(rt, txt_embeds, txt_masks, emb, masks, graph_sprels=self.graph_bias(graph_sprels))


class PreTrainedBase(nn.Module):
    """Stands in for transformers.BertPreTrainedModel: BERT weight init and a tolerant `from_pretrained`
    (the reference calls Cls.from_pretrained(None, config=cfg, state_dict=sd) with partial / superset
    state dicts, train_r2r.py:153-155)."""

    def __init__(self, config):
        super().__init__()
        self.config = config

    def init_weights(self):
        std = getattr(self.config, "initializer_range", 0.02)
        for m in self.modules():
            if isinstance(m, (nn.Linear, nn.Embedding)):
                m.weight.data.normal_(mean=0.0, std=std)
            elif isinstance(m, nn.LayerNorm):
                m.bias.data.zero_()
                m.weight.data.fill_(1.0)
            if isinstance(m, nn.Linear) and m.bias is not None:
                m.bias.data.zero_()

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path=None, config=None, state_dict=None, **kw):
        model = cls(config)
        if state_dict is not None:
            own = model.state_dict()
            keep = {k: v for k, v in state_dict.items() if k in own and own[k].shape == v.shape}
            model.load_state_dict(keep, strict=False)
        if hasattr(model, "tie_weights"):
            model.tie_weights()
        return model


class GlocalTextPathCMT(PreTrainedBase):  # :703-883
    def __init__(self, config):
        super().__init__(config)
        self.bev_dim = config.bev_dim
        self.embeddings = BertEmbeddings(config)
        self.lang_encoder = LanguageEncoder(config)
        self.img_embeddings = ImageEmbeddings(config)
        self.local_encoder = LocalBEVEncoder(config)
        self.global_encoder = GlobalMapEncoder(config)
        self.rt = Bk.Runtime()
        self._rt_external = False
        self.init_weights()

    # -- shared front ------------------------------------------------------------------------------
    def _begin(self):
        if not self._rt_external:          # a wrapper (pre-training model) may already have begun the step
            self.rt.feat_p = 0.0
            self.rt.begin(self.training)
        return self.rt

    def _front(self, rt, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
               traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens):
        txt_masks = gen_seq_masks(txt_lens, txt_ids.shape[1])
        txt = self.lang_encoder(rt, self.embeddings(rt, txt_ids), txt_masks)
        traj, traj_lens = self.img_embeddings(rt, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                                              traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens,
                                              self.embeddings.token_type_embeddings)
        return txt, txt_masks, traj, traj_lens

    def _last_obj_tokens(self, traj, traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens):
        """object tokens of each sample's last panorama (vilmodel.py:748-756) -> ((B,O,H), (B,O) bool)."""
        if traj_vp_obj_lens is None:
            return None, None
        dev = traj.device
        nP, Vtot, Hd = traj.shape
        last = torch.cumsum(torch.tensor(traj_step_lens, device=dev), 0) - 1
        vl, ol = traj_vp_view_lens[last], traj_vp_obj_lens[last]
        O = int(ol.max())
        ar = torch.arange(O, device=dev)[None, :]
        idx = torch.where(ar < ol[:, None], last[:, None] * Vtot + vl[:, None] + ar, torch.full_like(ar, -1))
        obj = Bk.run_block(Bk.GatherRowsImpl(), [traj.reshape(-1, Hd), idx.reshape(-1)], []).view(len(traj_step_lens), O, Hd)
        return obj, ar < ol[:, None]

    # -- public API (reference signatures) -----------------------------------------------------------
    def forward(self, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens,
                gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks,
                bev_nav_masks, return_gmap_embeds=True):
        rt = self._begin()
        txt, txt_masks, traj, traj_lens = self._front(rt, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts,
                                                      traj_loc_fts, traj_nav_types, traj_step_lens,
                                                      traj_vp_view_lens, traj_vp_obj_lens)
        gmap_embeds = None
        if return_gmap_embeds:
            gmap_embeds = self.global_encoder(rt, txt, txt_masks, traj, traj_lens, traj_step_lens, traj_vpids,
                                              traj_cand_vpids, gmap_vpids, gmap_step_ids, gmap_pos_fts, gmap_lens,
                                              graph_sprels=gmap_pair_dists)
        obj, obj_masks = self._last_obj_tokens(traj, traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens)
        bev_embeds, obj_embeds = self.local_encoder(rt, txt, txt_masks, bev_fts, bev_pos_fts, bev_masks,
                                                    bev_nav_masks, obj, obj_masks)
        return gmap_embeds, bev_embeds, obj_embeds, obj_masks

    def forward_mlm(self, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                    traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens,
                    gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks,
                    bev_nav_masks):
        rt = self._begin()
        txt, txt_masks, traj, traj_lens = self._front(rt, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts,
                                                      traj_loc_fts, traj_nav_types, traj_step_lens,
                                                      traj_vp_view_lens, traj_vp_obj_lens)
        tk = neg_key_mask(txt_masks)
        g_in, g_masks = self.global_encoder.gmap_input_embedding(
            rt, traj, traj_lens, traj_step_lens, traj_vpids, traj_cand_vpids, gmap_vpids, gmap_step_ids, gmap_pos_fts,
            gmap_lens)
        gk = neg_key_mask(g_masks)
        g_txt = txt
        for layer in self.global_encoder.encoder.x_layers:
            g_txt = layer.forward_lang2visn(rt, g_txt, tk, g_in, gk)
        obj, obj_masks = self._last_obj_tokens(traj, traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens)
        bev = self.local_encoder.bev_input_embedding(rt, bev_fts, bev_pos_fts, bev_nav_masks)
        if obj is not None:
            bev = torch.cat([bev, obj], dim=1)
            bev_masks = torch.cat([bev_masks, obj_masks], dim=1)
        bk = neg_key_mask(bev_masks)
        b_txt = txt
        for layer in self.local_encoder.encoder.x_layers:
            b_txt = layer.forward_lang2visn(rt, b_txt, tk, bev, bk)
        return Bk.run_block(Bk.AddRowsImpl(), [g_txt, b_txt, None], [None, None])

    def forward_sem(self, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts, traj_loc_fts, traj_nav_types,
                    traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens, traj_vpids, traj_cand_vpids, gmap_lens,
                    gmap_step_ids, gmap_pos_fts, gmap_pair_dists, gmap_vpids, bev_fts, bev_pos_fts, bev_masks,
                    bev_nav_masks, sem_pred_token=None):
        rt = self._begin()
        if sem_pred_token == "cattn":
            txt, txt_masks, traj, traj_lens = self._front(rt, txt_ids, txt_lens, traj_view_img_fts, traj_obj_img_fts,
                                                          traj_loc_fts, traj_nav_types, traj_step_lens,
                                                          traj_vp_view_lens, traj_vp_obj_lens)
            obj, obj_masks = self._last_obj_tokens(traj, traj_step_lens, traj_vp_view_lens, traj_vp_obj_lens)
            return self.local_encoder(rt, txt, txt_masks, bev_fts, bev_pos_fts, bev_masks, bev_nav_masks, obj,
                                      obj_masks)[0]
        bev = self.local_encoder.bev_input_embedding(rt, bev_fts, bev_pos_fts, bev_nav_masks)
        if sem_pred_token == "sattn":
            bk = neg_key_mask(bev_masks)
            for layer in self.local_encoder.encoder.x_layers:
                bev = layer.forward_visn2visn(rt, bev, bk)
        elif sem_pred_token != "embed":
            raise NotImplementedError
        return bev
