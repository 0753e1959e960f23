"""Oracle of the VLN-CE policy's `waypoint` call with in_train=False (bevbert_ce/vlnce_baselines/models/
Policy_ViewSelection_BEV.py:166-321) and of the trainer's _vp_feature_variable (ss_trainer_BEV.py:347-384), restated
with the reference's own torch operations over encoder callables passed in by the caller.  It runs wherever its inputs
live: on the CPU, or on the CUDA device with the reference's device arithmetic (the step's graph is compared with it).

`_vp_feature_variable` is restated rather than imported because its module imports habitat, lmdb and gym, which this
project does not depend on (as tests/ce_nav_bev_oracle.py restates the trainer's `splat`).
"""
import copy
import math

import numpy as np
import torch
import torch.nn.functional as F
from torch.nn.utils.rnn import pad_sequence

NUM_ANGLES, NUM_IMGS, NUM_CLASSES = 120, 12, 12


def angle_feature_torch(headings):
    return torch.stack([torch.sin(headings), torch.cos(headings), torch.sin(torch.zeros_like(headings)),
                        torch.cos(torch.zeros_like(headings))]).float().T


def pano_features():
    """BEV.__init__'s pano_img_idxes (12,) int64 and pano_angle_fts (12, 4)"""
    idx = np.arange(0, 12, dtype=np.int64)
    return idx, angle_feature_torch(torch.from_numpy((1 - idx / 12) * 2 * math.pi))


def waypoint_branch(observations, depth_encoder, rgb_encoder, waypoint_predictor, nms, pano_angle_fts, pano_img_idxes):
    """BEV.forward(mode='waypoint', in_train=False).  depth_encoder(obs) -> (12 B, 128, 4, 4); rgb_encoder(obs) ->
    ((12 B, 512), (12 B, 196, 768)); waypoint_predictor(rgb, depth) -> (B, 120, 12); nms as waypoint_pred/utils.py."""
    batch_size = observations['rgb'].shape[0]
    depth_batch = torch.zeros_like(observations['depth']).repeat(NUM_IMGS, 1, 1, 1)
    rgb_batch = torch.zeros_like(observations['rgb']).repeat(NUM_IMGS, 1, 1, 1)
    a_count = 0
    for k, v in observations.items():
        if 'depth' in k:
            for bi in range(v.size(0)):
                ra_count = (NUM_IMGS - a_count) % NUM_IMGS
                depth_batch[ra_count + bi * NUM_IMGS] = v[bi]
                rgb_batch[ra_count + bi * NUM_IMGS] = observations[k.replace('depth', 'rgb')][bi]
            a_count += 1
    obs_view12 = {'depth': depth_batch, 'rgb': rgb_batch}
    depth_embeds = depth_encoder(obs_view12)
    depth_grid_embeds = torch.flatten(F.adaptive_avg_pool2d(depth_batch.permute(0, 3, 1, 2), (14, 14)), 1)
    rgb_embeds, rgb_grid_embeds = rgb_encoder(obs_view12)
    logits = waypoint_predictor(rgb_embeds, depth_embeds)

    rgb_r = rgb_embeds.reshape(batch_size, NUM_IMGS, 512, 1, 1)
    rgb_feats = torch.cat([rgb_r[:, 0:1, :], torch.flip(rgb_r[:, 1:, :], [1])], dim=1)
    dep_r = depth_embeds.reshape(batch_size, NUM_IMGS, 128, 4, 4)
    depth_feats = torch.cat([dep_r[:, 0:1, :], torch.flip(dep_r[:, 1:, :], [1])], dim=1)
    rgb_grid_feats = rgb_grid_embeds.reshape(batch_size, NUM_IMGS, 196, 768)
    depth_grid_feats = depth_grid_embeds.reshape(batch_size, NUM_IMGS, 196, 1)

    x = torch.softmax(logits.reshape(batch_size, NUM_ANGLES * NUM_CLASSES), dim=1)
    x = x.reshape(batch_size, NUM_ANGLES, NUM_CLASSES)
    x = torch.cat((x[:, -1:, :], x, x[:, :1, :]), dim=1)
    out_map = nms(x.unsqueeze(1), max_predictions=5, sigma=(7.0, 5.0)).squeeze(1)[:, 1:-1, :]

    rgb_feats = torch.flatten(F.adaptive_avg_pool2d(rgb_feats, (1, 1)), 2)
    depth_feats = torch.flatten(F.adaptive_avg_pool2d(depth_feats, (1, 1)), 2)
    cand_rgb, cand_depth, cand_angle_fts, cand_img_idxes, cand_angles, cand_distances = [], [], [], [], [], []
    for j in range(batch_size):
        angle_idxes = out_map[j].nonzero()[:, 0]
        distance_idxes = out_map[j].nonzero()[:, 1]
        angle_rad_c = angle_idxes.cpu().float() / 120 * 2 * math.pi
        angle_rad_cc = 2 * math.pi - angle_idxes.float() / 120 * 2 * math.pi
        cand_angle_fts.append(angle_feature_torch(angle_rad_c))
        cand_angles.append(angle_rad_cc.tolist())
        cand_distances.append(((distance_idxes + 1) * 0.25).tolist())
        img_idxes = 12 - (angle_idxes.cpu().numpy() + 5) // 10
        img_idxes[img_idxes == 12] = 0
        cand_img_idxes.append(img_idxes)
        cand_rgb.append(rgb_feats[j, img_idxes, ...])
        cand_depth.append(depth_feats[j, img_idxes, ...])
    return {
        'cand_rgb': cand_rgb, 'cand_depth': cand_depth, 'cand_angle_fts': cand_angle_fts,
        'cand_img_idxes': cand_img_idxes, 'cand_angles': cand_angles, 'cand_distances': cand_distances,
        'pano_rgb': rgb_feats, 'pano_depth': depth_feats, 'pano_rgb_grid': rgb_grid_feats,
        'pano_depth_grid': depth_grid_feats, 'pano_angle_fts': copy.deepcopy(pano_angle_fts),
        'pano_img_idxes': copy.deepcopy(pano_img_idxes),
    }


def pad_tensors_wgrad(tensors):
    """vlnce_baselines/common/ops.py pad_tensors_wgrad: B x [T, ...] -> (B, max T, ...) zero-padded"""
    lens = [t.size(0) for t in tensors]
    max_len = max(lens)
    hid = list(tensors[0].size()[1:])
    out = []
    for t, n in zip(tensors, lens):
        if n < max_len:
            t = torch.cat([t, torch.zeros([max_len - n] + hid, dtype=t.dtype).to(t.device)], dim=0)
        out.append(t)
    return torch.stack(out, 0)


def vp_feature_variable(obs, device):
    """the trainer's _vp_feature_variable(obs) over len(obs['cand_angles']) environments; `.cuda()` is `.to(device)`"""
    batch_rgb_fts, batch_dep_fts, batch_loc_fts, batch_nav_types, batch_view_lens = [], [], [], [], []
    for i in range(len(obs['cand_angles'])):
        rgb_fts, dep_fts, loc_fts, nav_types = [], [], [], []
        cand_idxes = np.zeros(12, dtype=bool)
        cand_idxes[obs['cand_img_idxes'][i]] = True
        rgb_fts.append(obs['cand_rgb'][i])
        dep_fts.append(obs['cand_depth'][i])
        loc_fts.append(obs['cand_angle_fts'][i])
        nav_types += [1] * len(obs['cand_angles'][i])
        rgb_fts.append(obs['pano_rgb'][i][~cand_idxes])
        dep_fts.append(obs['pano_depth'][i][~cand_idxes])
        loc_fts.append(obs['pano_angle_fts'][~cand_idxes])
        nav_types += [0] * (12 - np.sum(cand_idxes))
        batch_rgb_fts.append(torch.cat(rgb_fts, dim=0))
        batch_dep_fts.append(torch.cat(dep_fts, dim=0))
        batch_loc_fts.append(torch.cat(loc_fts, dim=0))
        batch_nav_types.append(torch.LongTensor(nav_types))
        batch_view_lens.append(len(nav_types))
    return {'rgb_fts': pad_tensors_wgrad(batch_rgb_fts), 'dep_fts': pad_tensors_wgrad(batch_dep_fts),
            'loc_fts': pad_tensors_wgrad(batch_loc_fts).to(device),
            'nav_types': pad_sequence(batch_nav_types, batch_first=True).to(device),
            'view_lens': torch.LongTensor(batch_view_lens).to(device)}
