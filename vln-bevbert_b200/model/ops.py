"""Mask helpers and host-side index builders (reference: pretrain_src/model/ops.py:25-68 and the Python
loops of vilmodel.py:632-666 / pretrain_cmt.py:339-356, turned into index tensors built once per batch)."""
import torch

NEG_MASK = -10000.0


def gen_seq_masks(seq_lens, max_len=None):
    """(N,) lengths -> (N, max_len) bool (ops.py:36-44)."""
    if max_len is None:
        max_len = int(seq_lens.max())
    return torch.arange(max_len, device=seq_lens.device)[None, :] < seq_lens[:, None]


def neg_key_mask(masks, neg=NEG_MASK):
    """bool (N,L) -> additive fp32 (N,L): 0 where valid, `neg` where padded (extend_neg_masks, ops.py:25-34,
    without the broadcast dims -- the softmax kernel broadcasts over heads and queries)."""
    return (1.0 - masks.to(torch.float32)) * neg


def inf_key_mask(masks):
    """bool (N,L) valid -> additive fp32 with -inf on padding (nn.MultiheadAttention key_padding_mask)."""
    return torch.zeros(masks.shape, dtype=torch.float32, device=masks.device).masked_fill(~masks, float("-inf"))


def build_gmap_segments(traj_step_lens, traj_vp_lens, traj_vpids, traj_cand_vpids, gmap_vpids, G, Vtot, device):
    """CSR lists for the topological-map node features (vilmodel.py:632-666).

    Node j of sample i (row i*G + j) is
      - the mean over the valid tokens of the panorama of a visited viewpoint, or
      - the mean of the candidate-view tokens (over all panoramas) that point at an unvisited viewpoint;
    row j = 0 ([stop]) and padded rows are empty segments (zeros).  Token (pano p, view v) is row p*Vtot+v of
    the flattened panorama embeddings.  The lists come from host strings only; the per-panorama token counts
    (`traj_vp_lens`, a device tensor) enter through the weights, which are finished on the device
    (w = [v < len] / len for visited nodes) -- so building them never synchronises with the GPU.
    """
    seg_off, idx, w, wpano = [0], [], [], []
    p0 = 0
    for i, P in enumerate(traj_step_lens):
        visited_at = {}
        cand_tok = {}
        for t in range(P):
            visited_at[traj_vpids[i][t]] = p0 + t
            for j, vp in enumerate(traj_cand_vpids[i][t]):
                if vp not in visited_at:
                    cand_tok.setdefault(vp, []).append((p0 + t) * Vtot + j)
        nodes = gmap_vpids[i]
        for j in range(G):
            if 0 < j < len(nodes):
                vp = nodes[j]
                if vp in visited_at:
                    pano = visited_at[vp]
                    idx.extend(range(pano * Vtot, (pano + 1) * Vtot))
                    w.extend([0.0] * Vtot)               # filled on the device from the token counts
                    wpano.extend([pano] * Vtot)
                else:
                    toks = cand_tok[vp]
                    idx.extend(toks)
                    w.extend([1.0 / len(toks)] * len(toks))
                    wpano.extend([-1] * len(toks))
            seg_off.append(len(idx))
        p0 += P
    host = torch.tensor([idx, wpano], dtype=torch.int32)
    wh = torch.tensor(w, dtype=torch.float32)
    so = torch.tensor(seg_off, dtype=torch.int32)
    return finish_gmap_segments((host, wh, so), traj_vp_lens, Vtot, device)


def host_gmap_segments(traj_step_lens, traj_vpids, traj_cand_vpids, gmap_vpids, G, Vtot):
    """The host half of build_gmap_segments (string matching only) -- can run in the data loader / collate."""
    seg = build_gmap_segments(traj_step_lens, None, traj_vpids, traj_cand_vpids, gmap_vpids, G, Vtot, None)
    return seg


def finish_gmap_segments(host_parts, traj_vp_lens, Vtot, device):
    """Device half: upload the host lists (pinned, non-blocking) and finish the visited-node weights from the
    per-panorama token counts."""
    host, wh, so = host_parts
    if device is None:
        return host_parts
    if device.type == "cuda":
        host, wh, so = [t if t.is_pinned() else t.pin_memory() for t in (host, wh, so)]
    dv = host.to(device, non_blocking=True)
    wd = wh.to(device, non_blocking=True)
    idx_d, pano_d = dv[0].contiguous(), dv[1].long()
    lens = traj_vp_lens.to(torch.float32)
    vis = pano_d >= 0
    pc = pano_d.clamp(min=0)
    view = (idx_d.long() - pc * Vtot).to(torch.float32)
    w_vis = (view < lens[pc]).to(torch.float32) / lens[pc]
    return so.to(device, non_blocking=True), idx_d, torch.where(vis, w_vis, wd)


class PreparedList(list):
    """A host id list that carries index tensors precomputed from it (see prepare_batch)."""
    host_segments = None
    host_fusion = None
    host_mlm = None


WIRE_KEYS = ("rgbs", "traj_view_img_fts", "traj_view_dep_fts", "traj_obj_img_fts")


def prepare_batch(batch, wire_dtype=None):
    """Optional collate-time step (the reference's `sap_collate` / `mlm_collate` run in DataLoader workers,
    pretrain_src/data/tasks.py:118-160): does the string matching behind the topological-map aggregation and the
    SAP logit fusion once, on the host, into pinned index tensors attached to `batch['gmap_vpids']`.  forward()
    finds and uses them; without this call it builds the same tensors itself (same results, more host time
    inside the step).  `wire_dtype=torch.bfloat16` additionally converts the large fp32 feature tensors (WIRE_KEYS)
    to bf16 on the host; the model accepts either dtype."""
    gv = PreparedList(batch["gmap_vpids"])
    G = batch["gmap_step_ids"].shape[1]
    Vtot = batch["traj_loc_fts"].shape[1]
    parts = host_gmap_segments(batch["traj_step_lens"], batch["traj_vpids"], batch["traj_cand_vpids"], gv, G, Vtot)
    pin = torch.cuda.is_available()
    gv.host_segments = ((G, Vtot), tuple(t.pin_memory() if pin else t for t in parts))
    if "bev_cand_idxs" in batch:
        Kc = batch["bev_cand_idxs"].shape[1]
        E2 = _fusion_matches(gv, [c[-1] for c in batch["traj_cand_vpids"]], G, Kc)
        gv.host_fusion = ((G, Kc), E2.pin_memory() if pin else E2)
    lab = batch.get("txt_labels")
    if torch.is_tensor(lab) and not lab.is_cuda:
        # masked-token rows and their labels (pretrain_cmt.py:259-270 selects them with a boolean mask on the device,
        # which costs a device->host sync per MLM step); the masking was drawn on the host, so the list is known here
        flat = lab.reshape(-1)
        idx = torch.nonzero(flat != -1, as_tuple=False).reshape(-1)
        sel = flat[idx].contiguous()
        gv.host_mlm = (tuple(lab.shape), idx.pin_memory() if pin else idx, sel.pin_memory() if pin else sel)
    out = dict(batch)
    out["gmap_vpids"] = gv
    if wire_dtype is not None:
        # 16-bit wire format for the large feature tensors (the grid / view features are stored as 16-bit floats in the
        # reference's HDF5 files and are bf16 GEMM operands on the device): halves the host->device bytes per step
        for k in WIRE_KEYS:
            v = out.get(k)
            if torch.is_tensor(v) and v.dtype == torch.float32:
                v = v.to(wire_dtype)
                out[k] = v.pin_memory() if pin else v
        # semantic labels: the float64 one-hots of dataset.py:402 back to the uint8 class ids they were built from
        # (lossless when every row is exactly one-hot, which is how the reference constructs them)
        sem = out.get("sems")
        if torch.is_tensor(sem) and sem.dtype == torch.float64 and sem.dim() == 3 and sem.shape[-1] <= 64:
            ids = sem.argmax(-1)
            if bool((sem.sum(-1) == 1).all()) and bool((sem.gather(-1, ids[..., None]) == 1).all()):
                ids = ids.to(torch.uint8)
                out["sems"] = ids.pin_memory() if pin else ids
    return out


def _fusion_matches(gmap_vpids, last_cand_vpids, G, Kc, out=None):
    """(2,B,G,Kc) host matrix: [0] every (node j == candidate k) match, [1] only the last candidate per viewpoint.
    `out`: an fp32 host tensor of that shape to fill instead of a new one (a pinned staging buffer)."""
    B = len(gmap_vpids)
    E2 = torch.zeros(2, B, G, Kc, dtype=torch.float32) if out is None else out.zero_()
    e = E2.numpy()                                        # element writes through numpy: no torch op per match
    for i in range(B):
        pos = {vp: j for j, vp in enumerate(gmap_vpids[i]) if j > 0}
        last = {}
        for k, vp in enumerate(last_cand_vpids[i]):
            j = pos.get(vp)
            if j is not None and k + 1 < Kc:
                e[0, i, j, k + 1] = 1.0
                last[vp] = (j, k + 1)                     # `tmp[cand_vpid] = ...` overwrites: the last view wins
        for j, k in last.values():
            e[1, i, j, k] = 1.0
    return E2


def build_sap_fusion(gmap_vpids, gmap_visited_masks, last_cand_vpids, G, Kc, device):
    """(B, G, Kc) 0/1 fp32 matrix F with fused[b,j] = global[b,j] + sum_k F[b,j,k] * local[b,k]
    (pretrain_cmt.py:339-356): slot 0 takes local[0]; an unvisited node takes the local logit of the
    candidate view that reaches it, otherwise the sum over candidates that lead back to visited nodes.
    The viewpoint-id matching E[b,j,k] = (node j is candidate k) is host string work; whether a node is
    visited comes from the device mask, so F is finished on the device without a host synchronisation."""
    B = len(gmap_vpids)
    pre = getattr(gmap_vpids, "host_fusion", None)
    E2 = pre[1] if (pre is not None and pre[0] == (G, Kc)) else _fusion_matches(gmap_vpids, last_cand_vpids, G, Kc)
    if device.type == "cuda" and not E2.is_pinned():
        if torch.cuda.is_current_stream_capturing():
            # a graph would re-read this temporary host buffer at every replay, long after it was freed
            raise RuntimeError("build_sap_fusion under CUDA-graph capture needs the fusion matches staged in a pinned "
                               "buffer (PreparedList.host_fusion)")
        E2 = E2.pin_memory()
    E2 = E2.to(device, non_blocking=True)
    vis = gmap_visited_masks.to(torch.float32)                     # (B,G)
    cand_visited = torch.einsum("bgk,bg->bk", E2[0], vis)          # candidate k leads back to a visited node
    direct = E2[1] * (1.0 - vis)[:, :, None]                       # unvisited node j reached by candidate k
    has_direct = direct.sum(2, keepdim=True) > 0
    unvis = (1.0 - vis)
    unvis[:, 0] = 0.0                                              # slot 0 handled separately
    F = torch.where(has_direct, direct, cand_visited[:, None, :].expand(B, G, Kc)) * unvis[:, :, None]
    # padded gmap slots (beyond gmap_len) have no vpid: they only ever get the back-logit term, like the reference
    F[:, 0, :] = 0.0
    F[:, 0, 0] = 1.0
    return F


# ------------------------------------------------------------------ reference-named helpers (drop-in surface)
def extend_neg_masks(masks, dtype=None):
    """(N, L) bool -> (N, 1, 1, L) additive mask, 0 where valid and -10000 where padded
    (pretrain_src/model/ops.py:25-34, map_nav_src/models/ops.py:25-34).  The kernels take the (N, L) form
    (`neg_key_mask`); this is the reference's broadcastable shape for callers that build masks themselves."""
    return neg_key_mask(masks).to(dtype or torch.float32)[:, None, None, :]


def pad_tensors_wgrad(tensors, lens=None):
    """B x [T_i, ...] -> (B, max T, ...) zero-padded, gradients flow to the inputs (pretrain_src/model/ops.py:46-68,
    map_nav_src/models/ops.py:46-68; used by map_nav_src/r2r/agent.py:250, reverie/agent_obj.py:254,345).
    One allocation + B slice copies instead of a cat per sample."""
    if lens is None:
        lens = [t.size(0) for t in tensors]
    max_len = max(lens)
    out = tensors[0].new_zeros((len(tensors), max_len) + tuple(tensors[0].shape[1:]))
    if any(t.requires_grad for t in tensors):
        parts = []
        for t, n in zip(tensors, lens):
            parts.append(t if n == max_len else torch.cat([t, t.new_zeros((max_len - n,) + tuple(t.shape[1:]))], 0))
        return torch.stack(parts, 0)
    for i, (t, n) in enumerate(zip(tensors, lens)):
        out[i, :n] = t[:n]
    return out
