"""Point-cloud normalisation used by the scores (reference utils/data_helper.py:9-35)."""


def normalize_point_clouds(pcs, mode='shape_bbox'):
    """Centre every cloud on its bounding-box centre and scale it so that the longest box side spans [-1, 1].

    pcs: a list of [N,C] tensors or a [B,N,C] tensor, C in (3, 4, 6, 9); only the first three channels are moved.
    Returns a list of new tensors; the input is not modified."""
    assert isinstance(pcs, list) or len(pcs.shape) == 3, f'expect pcs to be list, get: {type(pcs)} or 3d tensor; '
    assert mode == 'shape_bbox'
    out = []
    for i in range(len(pcs)):
        pc = pcs[i].detach().clone()
        assert len(pc.shape) == 2 and pc.shape[-1] in (3, 4, 6, 9), f'expect get (N,3 or 6), get {pc.shape}'
        hi = pc.max(dim=0, keepdim=True)[0][:, :3]
        lo = pc.min(dim=0, keepdim=True)[0][:, :3]
        shift = ((lo + hi) / 2).view(1, 3)
        scale = (hi - lo).max().reshape(1, 1) / 2
        pc[:, :3] = (pc[:, :3] - shift) / scale
        out.append(pc)
    return out
