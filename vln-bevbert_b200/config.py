"""Model configuration: the HF-style attribute bag the reference's model classes read
(configs/r2r_model.json + the attributes bolted on at pretrain_src/train_r2r.py:102-105; SURVEY.md 5)."""
from types import SimpleNamespace

R2R_DEFAULTS = dict(
    hidden_size=768, num_attention_heads=12, intermediate_size=3072, hidden_act="gelu",
    hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, layer_norm_eps=1e-12,
    vocab_size=30522, max_position_embeddings=512, type_vocab_size=2, initializer_range=0.02,
    num_l_layers=9, num_x_layers=4, num_pano_layers=2, num_hidden_layers=12,
    image_feat_size=768, angle_feat_size=4, obj_feat_size=0, obj_prob_size=0, max_action_steps=100,
    update_lang_bert=True, use_lang2visn_attn=True, graph_sprels=True, glocal_fuse=True,
    bev_dim=21, bev_res=0.5, feat_dropout=0.4, output_attentions=False, output_hidden_states=False,
    pretrain_tasks=["mlm", "sap", "masksem"], sem_pred_token="cattn",
)

# VLN-CE pre-training (bevbert_ce/pretrain/run_pt/r2r_model_config_dep.json; tasks of r2r_pretrain_habitat.json):
# 512-d CLIP view features, 128-d depth features, 4 angle columns, no objects, an 11 x 11 BEV at 1 m
CE_DEFAULTS = dict(R2R_DEFAULTS, image_feat_size=512, depth_feat_size=128, image_prob_size=1000, bev_dim=11, bev_res=1.0,
                   pretrain_tasks=["mlm", "sap"])
# a 2/1/2-layer CE model with dropout off: the parity tests' and smoke runs' size
CE_SMALL = dict(num_l_layers=2, num_x_layers=2, num_pano_layers=1, vocab_size=3000, hidden_dropout_prob=0.0,
                attention_probs_dropout_prob=0.0, feat_dropout=0.0)


# VLN-CE navigation (bevbert_ce/vlnce_baselines/models/bev/vlnbert_init.py:35-59 over bert-base-uncased): the keys
# get_vlnbert_models sets, with depth embedding and graph sprels on (the R2R-CE run configs)
CE_NAV_DEFAULTS = dict(R2R_DEFAULTS, image_feat_size=512, use_depth_embedding=True, depth_feat_size=128,
                       angle_feat_size=4, graph_sprels=True, glocal_fuse="dynamic", fix_lang_embedding=False,
                       fix_pano_embedding=False, output_attentions=True, pred_head_dropout_prob=0.1,
                       use_lang2visn_attn=False, bev_dim=11, bev_res=1.0)


def make_config(**overrides):
    """Returns a transformers.PretrainedConfig when transformers is importable (what the reference's
    BertPreTrainedModel subclasses need), else a SimpleNamespace with the same attributes."""
    vals = dict(R2R_DEFAULTS)
    vals.update(overrides)
    try:
        from transformers import PretrainedConfig
        cfg = PretrainedConfig()
        for k, v in vals.items():
            setattr(cfg, k, v)
        return cfg
    except Exception:  # pragma: no cover
        return SimpleNamespace(**vals)


def make_ce_config(small=False, **overrides):
    """make_config for the VLN-CE model (model/ce_pretrain.py); `small` applies CE_SMALL before `overrides`."""
    vals = dict(CE_DEFAULTS)
    if small:
        vals.update(CE_SMALL)
    vals.update(overrides)
    return make_config(**vals)


def make_ce_nav_config(small=False, **overrides):
    """make_config for the VLN-CE navigation network (model/ce_nav.py); `small` applies CE_SMALL before `overrides`.
    The reference's `use_sprels` is `graph_sprels` here, as in vlnbert_init.py."""
    vals = dict(CE_NAV_DEFAULTS)
    if small:
        vals.update(CE_SMALL)
    vals.update(overrides)
    return make_config(**vals)
