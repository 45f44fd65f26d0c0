"""Host-side mirror of the reference's ARAP regulariser (custom/threestudio-animate3d/systems/util.py:58-117, 138-215;
called from systems/animate3d.py:215-244), on the CUDA path of liba3d.so:

    ii, jj, nn, weight = cal_connectivity_from_points(points, radius=..., K=...)
    loss_arap = cal_arap_error(nodes_t, ii, jj, nn, K=..., sample_num=...)

`cal_connectivity_from_points` supports the mode every shipped config uses ('nn', adaptive weighting); the KNN graph comes
from `a3d_knn_graph`.  `cal_arap_error` runs the fused rotation-fit + energy + gradient kernel (`a3d_arap`) for all frames
at once and is differentiable w.r.t. the node positions (the rotation itself carries no gradient, as in the reference).
Under torch.use_deterministic_algorithms(True) it sums energy and gradient in a fixed order."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib as L


def knn_graph(points: torch.Tensor, K: int):
    """[Nv,3] cuda fp32 -> (nbr [Nv,K] int32, dist2 [Nv,K]) of the K nearest other points (squared distances, ascending)."""
    lib = L.load()
    pts = points.detach().contiguous().float()
    n = pts.shape[0]
    nbr = torch.empty(n, K, dtype=torch.int32, device=pts.device)
    d2 = torch.empty(n, K, dtype=torch.float32, device=pts.device)
    L.check(lib.a3d_knn_graph(C.c_void_p(pts.data_ptr()), n, K, C.c_void_p(nbr.data_ptr()), C.c_void_p(d2.data_ptr()), L.stream_ptr()))
    return nbr, d2


def cal_connectivity_from_points(points: torch.Tensor, radius: float = 0.1, K: int = 10, least_edge_num: int = 3):
    """util.py:58-117, mode 'nn', adaptive_weighting=True.  points [Nt,Nv,3] (frame 0 defines the graph).  Returns
    (ii, jj, nn, weight) exactly like the reference."""
    nv = points.shape[1]
    nbr, nn_dist = knn_graph(points[0], K)
    nn_idx = nbr.long()
    if points.shape[0] > 1:
        rest = points[1:][:, nn_idx]
        rest_d = ((rest - points[0:1][:, :, None]) ** 2).sum(-1)
        nn_dist = torch.where((rest_d < radius ** 2).all(0), nn_dist, torch.full_like(nn_dist, float("inf")))
    far = nn_dist[:, least_edge_num:] >= radius ** 2
    nn_idx[:, least_edge_num:] = torch.where(far, torch.full_like(nn_idx[:, least_edge_num:], -1), nn_idx[:, least_edge_num:])
    nn_dist = nn_dist.clone()
    nn_dist[:, least_edge_num:] = torch.where(far, torch.full_like(nn_dist[:, least_edge_num:], float("inf")), nn_dist[:, least_edge_num:])
    weight = torch.exp(-nn_dist / nn_dist.mean())
    weight = weight / weight.sum(dim=-1, keepdim=True)
    dev = points.device
    ii = torch.arange(nv, device=dev)[:, None].expand(nv, K).reshape(-1)
    jj = nn_idx.reshape(-1)
    nn = torch.arange(K, device=dev)[None].expand(nv, K).reshape(-1)
    return drop_missing_edges(ii, jj, nn) + (weight,)


def drop_missing_edges(ii, jj, nn):
    """The edges with jj != -1.  The boolean selection reads its count from the device, so inside a CUDA-graph capture the
    full lists are returned: cal_arap_error writes their -1 entries into the table's -1 fill, which gives the same table."""
    if torch.cuda.is_current_stream_capturing():
        return ii, jj, nn
    keep = jj != -1
    return ii[keep], jj[keep], nn[keep]


def sample_nodes(nv: int, sample_num: int, device) -> torch.Tensor:
    """`sample_num` node indices drawn uniformly with replacement (the distribution of np.random.choice(nv, sample_num)) from
    torch's CUDA generator, whose draws a CUDA graph replays with a fresh offset each time."""
    return torch.randint(0, nv, (sample_num,), device=device)


last_sample_idx: Optional[torch.Tensor] = None    # the node sample of the most recent cal_arap_error (None: all nodes)


class _Arap(torch.autograd.Function):
    @staticmethod
    def forward(ctx, nodes, nbr, weight, sample):
        lib = L.load()
        x = nodes.detach().contiguous().float()
        nt, nv, _ = x.shape
        err = torch.empty(1, device=x.device)
        grad = torch.empty_like(x)
        k, ns = nbr.shape[1], nv if sample is None else sample.numel()
        det = L.deterministic()
        nbytes = lib.a3d_arap_scratch_bytes(nt, nv, k, ns, det)
        scratch = L.scratch(nbytes, x.device)
        L.check(lib.a3d_arap(C.c_void_p(x.data_ptr()), nt, nv, C.c_void_p(nbr.data_ptr()), k, C.c_void_p(L.ptr(weight)),
                             C.c_void_p(L.ptr(sample)), ns, det, C.c_void_p(err.data_ptr()), C.c_void_p(grad.data_ptr()),
                             C.c_void_p(L.ptr(scratch)), C.c_size_t(nbytes), L.stream_ptr()))
        ctx.save_for_backward(grad)
        return err[0]

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None, None, None


def cal_arap_error(nodes_sequence: torch.Tensor, ii, jj, nn, K: int = 10, weight: Optional[torch.Tensor] = None,
                   sample_num: int = 512, sample_idx: Optional[torch.Tensor] = None) -> torch.Tensor:
    """util.py:183-215.  nodes_sequence [Nt,Nv,3]; (ii, jj, nn) the edge list of `cal_connectivity_from_points`;
    weight [Nv,K] or None (1 on existing edges).  When Nv > sample_num a random node subset is drawn with
    np.random.choice(Nv, sample_num) like the reference (pass `sample_idx` to fix it); inside a CUDA-graph capture it is
    drawn on the device by `sample_nodes`.  `last_sample_idx` holds the sample used."""
    global last_sample_idx
    nt, nv, _ = nodes_sequence.shape
    dev = nodes_sequence.device
    nbr = torch.full((nv, K), -1, dtype=torch.int32, device=dev)
    nbr[ii, nn] = jj.to(torch.int32)
    if sample_idx is None and nv > sample_num:
        if torch.cuda.is_current_stream_capturing():
            sample_idx = sample_nodes(nv, sample_num, dev)
        else:
            sample_idx = torch.from_numpy(np.random.choice(nv, sample_num)).to(dev)
    s = None if sample_idx is None else sample_idx.to(device=dev, dtype=torch.int32).contiguous()
    last_sample_idx = s
    w = None if weight is None else weight.detach().contiguous().float()
    return _Arap.apply(nodes_sequence, nbr, w, s)
