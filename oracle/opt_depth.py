"""TEST INFRASTRUCTURE ONLY — the two geometric loss blocks of MultiplyModel.opt_depth restated, parameterised by the
three operators they call, so the same lines run on the float64 definitions (oracle/raster.py, oracle/mesh_port.py,
oracle/port.py) and on the device drop-ins (multiply_b200.model.render.Renderer, utils.kaolin_ops.check_sign,
utils.pytorch3d_ops.knn_points).  tests/golden/opt_depth.npz pins both blocks against the reference's own code
(oracle/gen_golden_opt_depth.py).

All ``file:line`` cites are relative to /root/reference/code.
"""
import torch


def interpenetration_loss(vertex_list, face_list, check_sign, knn_points, perms, num_pixels=5120):
    """MultiplyModel.get_interpenetration_loss (multiply_model.py:521-551).  vertex_list [1,V_p,3], face_list [F_p,3]
    or [1,F_p,3]; perms[p] = the draw of ``torch.randperm(vertex.shape[1])`` for person p (:526)."""
    loss = torch.zeros(1, device=vertex_list[0].device, dtype=vertex_list[0].dtype)        # :523
    for person_id, vertex in enumerate(vertex_list):
        idx = perms[person_id][:num_pixels].to(vertex.device)                                 # :526
        sample_point = torch.index_select(vertex, dim=1, index=idx)                           # :527
        for partner_id in range(len(vertex_list)):
            if partner_id == person_id:
                continue
            sign = check_sign(vertex_list[partner_id], face_list[partner_id].reshape(-1, 3),
                              sample_point).to(vertex.dtype)                                  # :532-534
            sign = sign.squeeze(0)
            sign = 1 - 2 * sign                                                               # :535-536
            if (sign < 0).any():
                penetrate_point = sample_point[:, sign < 0]
                _, _, neighbor_points = knn_points(penetrate_point, vertex_list[partner_id], K=1, return_nn=True)
                neighbor_points = neighbor_points.mean(dim=2)                                 # :543
                stable_point = (penetrate_point - neighbor_points).norm(dim=-1).reshape(-1) < 0.1   # :545
                if stable_point.any():
                    penetrate_point = penetrate_point.reshape(-1, 3)[stable_point]
                    neighbor_points = neighbor_points.reshape(-1, 3)[stable_point]
                    loss = loss + torch.nn.functional.mse_loss(penetrate_point, neighbor_points, reduction="sum")
    return loss


def depth_order_loss(depth_maps, sam_logits, max_depth=999):
    """The depth-order block of opt_depth (multiply_model.py:399-475) without its weights: depth_maps = the renderer's
    per-person [1,H,W,1] maps (layer 0, :399-401), sam_logits [1,H,W,P] = inputs["org_sam_mask"] (:415).  Returns
    (sum log(1 + exp(gt - front)) over the valid pixels where gt != front, or None where the reference takes the
    exclude_mask.sum() == 0 branch (:462-466), and the number of such pixels).  The caller applies depth_order_weight
    and the epoch ramp (:470-472)."""
    reshape_depth_map_list = [d[0, :, :, 0] for d in depth_maps]                              # :399-401
    max_depth_map_list = []
    for depth_map_i in reshape_depth_map_list:                                                # :404-411
        depth_map_processed = depth_map_i.clone()
        no_interaction = depth_map_processed < 0
        depth_map_processed[no_interaction] = max_depth
        max_depth_map_list.append(depth_map_processed)
    max_depth_map = torch.stack(max_depth_map_list, dim=-1)                                   # :412
    front_depth_map, _ = torch.min(max_depth_map, dim=-1)                                     # :413
    valid_mask = front_depth_map < max_depth                                                  # :414
    sam_mask = torch.sigmoid(sam_logits).squeeze(0)                                           # :415-418
    valid_mask = torch.logical_and(valid_mask, sam_mask.sum(dim=-1) <= (1 + 1e-2))            # :420
    valid_mask = torch.logical_and(valid_mask, sam_mask.sum(dim=-1) >= 0.7)                   # :421
    sam_mask_idx = torch.argmax(sam_mask, dim=-1).unsqueeze(-1)                               # :423-427
    gt_depth_map = torch.gather(max_depth_map, dim=-1, index=sam_mask_idx).squeeze(-1)        # :428-429
    valid_mask = torch.logical_and(valid_mask, gt_depth_map < max_depth)                      # :430
    valid_mask = valid_mask.flatten()                                                         # :453-455
    gt_depth_map = gt_depth_map.flatten()[valid_mask]
    front_depth_map = front_depth_map.flatten()[valid_mask]
    exclude_mask = ~(gt_depth_map == front_depth_map)                                         # :456
    n = int(exclude_mask.sum())
    if n == 0:
        return None, 0
    loss = torch.log(1 + torch.exp(gt_depth_map[exclude_mask] - front_depth_map[exclude_mask])).sum()   # :469
    return loss, n
