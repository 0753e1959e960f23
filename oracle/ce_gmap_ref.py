"""Restatement of the VLN-CE trainer's global-map image glue (bevbert_ce/vlnce_baselines): the rollout's masked mean and
candidate rows (ss_trainer_BEV.py:1032-1033, 1060-1066), the embedding half of GraphMap.update_graph / delete_ghost /
get_node_embeds (models/graph_utils.py:168-281) and _nav_gmap_variable's stack and pad_tensors_wgrad (ss_trainer_BEV.py:
534-611, common/ops.py:46-68).  Positions are (x, y, z) numpy arrays, as the trainer's are; everything else about the
graph (edges, shortest paths, ghost_aug positions) is out of this restatement's scope."""
import numpy as np
import torch


class GraphMap:
    """graph_utils.GraphMap's node / ghost bookkeeping and embeddings"""

    def __init__(self, has_real_pos, loc_noise, merge_ghost, ghost_aug):
        """the reference's constructor; has_real_pos and ghost_aug only move positions, which are out of scope here"""
        self.loc_noise, self.merge_ghost = loc_noise, merge_ghost
        self.node_pos, self.node_embeds, self.node_stepId = {}, {}, {}
        self.ghost_cnt = 0
        self.ghost_pos, self.ghost_mean_pos, self.ghost_embeds, self.ghost_fronts = {}, {}, {}, {}

    def _localize(self, qpos, kpos_dict):
        min_dis, min_vp = 10000, None
        for kvp, kpos in kpos_dict.items():
            dis = ((qpos - kpos) ** 2).sum() ** 0.5
            if dis < min_dis:
                min_dis, min_vp = dis, kvp
        return None if min_dis > self.loc_noise else min_vp

    def delete_ghost(self, vp):
        for d in (self.ghost_pos, self.ghost_mean_pos, self.ghost_embeds, self.ghost_fronts):
            d.pop(vp)

    def update_graph(self, prev_vp, step_id, cur_vp, cur_pos, cur_embeds, cand_vp, cand_pos, cand_embeds,
                     cand_real_pos):
        self.node_pos[cur_vp] = cur_pos
        self.node_embeds[cur_vp] = cur_embeds
        self.node_stepId[cur_vp] = step_id
        for cvp, cpos, cembeds in zip(cand_vp, cand_pos, cand_embeds):
            if self._localize(cpos, self.node_pos) is not None:
                continue
            gvp = self._localize(cpos, self.ghost_mean_pos) if self.merge_ghost else None
            if gvp is None:
                gvp = "g%d" % self.ghost_cnt
                self.ghost_cnt += 1
                self.ghost_pos[gvp] = [cpos]
                self.ghost_mean_pos[gvp] = cpos
                self.ghost_embeds[gvp] = [cembeds, 1]
                self.ghost_fronts[gvp] = [cur_vp]
            else:
                self.ghost_pos[gvp].append(cpos)
                self.ghost_mean_pos[gvp] = np.mean(self.ghost_pos[gvp], axis=0)
                self.ghost_embeds[gvp][0] = self.ghost_embeds[gvp][0] + cembeds
                self.ghost_embeds[gvp][1] += 1
                self.ghost_fronts[gvp].append(cur_vp)

    def get_node_embeds(self, vp):
        if not vp.startswith("g"):
            return self.node_embeds[vp]
        return self.ghost_embeds[vp][0] / self.ghost_embeds[vp][1]


def pad_tensors_wgrad(tensors):
    max_len = max(t.size(0) for t in tensors)
    hid = list(tensors[0].size()[1:])
    out = [torch.cat([t, torch.zeros([max_len - t.size(0)] + hid, dtype=t.dtype).to(t.device)], 0)
           if t.size(0) < max_len else t for t in tensors]
    return torch.stack(out, 0)


def update_graphs(gmaps, step_id, pano_embeds, pano_masks, nav_types, cur_vp, cur_pos, cand_vp, cand_pos):
    """the rollout's lines 1032-1033 and 1060-1066 (cand_real_pos None)"""
    avg_pano_embeds = torch.sum(pano_embeds * pano_masks.unsqueeze(2), 1) / torch.sum(pano_masks, 1, keepdim=True)
    for i, gmap in enumerate(gmaps):
        cand_embeds = pano_embeds[i][nav_types[i] == 1]
        gmap.update_graph(None, step_id, cur_vp[i], cur_pos[i], avg_pano_embeds[i], cand_vp[i], cand_pos[i],
                          cand_embeds, None)


def gmap_img_fts(gmaps):
    """_nav_gmap_variable's gmap_img_fts"""
    fts = []
    for gmap in gmaps:
        rows = [gmap.get_node_embeds(vp) for vp in gmap.node_pos] + [gmap.get_node_embeds(vp) for vp in gmap.ghost_pos]
        fts.append(torch.stack([torch.zeros_like(rows[0])] + rows, 0))
    return pad_tensors_wgrad(fts)
