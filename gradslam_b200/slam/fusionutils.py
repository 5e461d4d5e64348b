"""PointFusion map update: projective data association + confidence-weighted surfel fusion.

Host-side mirror of gradslam/slam/fusionutils.py (same function names, arguments, return types, errors and
warnings).  `update_map_fusion` runs as two hand-written sm_90a kernels over an in-place, capacity-backed
map (csrc/gsx_fusion.cu): no table is materialised, no whole-map clone / cat per frame, no host sync.  The
table-returning helpers (`find_active_map_points`, `find_similar_map_points`,
`find_best_unique_correspondences`, `fuse_with_map`) are kept for API parity and run the same arithmetic
through the table kernels in csrc/gsx_tables.cu.
"""
import math
import threading
import warnings
from typing import Union

import torch

from .. import _C
from ..structures.pointclouds import EMBED_DTYPES, Pointclouds, _PruneHistory
from ..structures.rgbdimages import RGBDImages, _frame_base

__all__ = ["update_map_fusion", "update_map_aggregate", "prune_unstable", "fuse_and_prune"]


# --------------------------------------------------------------------------------------------- small helpers
def get_alpha(points: torch.Tensor, sigma: Union[torch.Tensor, float, int], dim: int = -1, keepdim: bool = False,
              eps: float = 1e-7) -> torch.Tensor:
    """Sample confidence alpha = clamp(exp(-|p|^2 / 2 sigma^2), eps, 1.01) (fusionutils.py:16-73).
    Differentiable torch helper; inside the fused update alpha is evaluated by the merge kernel."""
    if not torch.is_tensor(points):
        raise TypeError("Expected input points to be of type torch.Tensor. Got {0} instead.".format(type(points)))
    if not (torch.is_tensor(sigma) or isinstance(sigma, (float, int))):
        raise TypeError("Expected input sigma to be of type torch.Tensor or float or int. Got {0} instead.".format(
            type(sigma)))
    if not isinstance(eps, float):
        raise TypeError("Expected input eps to be of type float. Got {0} instead.".format(type(eps)))
    if points.shape[dim] != 3:
        raise ValueError("Expected length of dim-th ({0}th) dimension to be 3. Got {1} instead.".format(
            dim, points.shape[dim]))
    if torch.is_tensor(sigma) and sigma.ndim != 0:
        raise ValueError("Expected sigma.ndim to be 0 (scalar). Got {0}.".format(sigma.ndim))
    sq = torch.sum(points ** 2, dim, keepdim=keepdim)
    return torch.clamp(torch.exp(-sq / (2 * (sigma ** 2))), min=eps, max=1.01)


def _pair_checks(tensor1, tensor2, th, th_name, dim):
    for name, t in (("tensor1", tensor1), ("tensor2", tensor2)):
        if not torch.is_tensor(t):
            raise TypeError("Expected input {} to be of type torch.Tensor. Got {} instead.".format(name, type(t)))
    if not isinstance(th, (float, int)):
        raise TypeError("Expected input {} to be of type float or int. Got {} instead.".format(th_name, type(th)))
    if tensor1.shape != tensor2.shape:
        raise ValueError("tensor1 and tensor2 should have the same shape, but had shapes {0} and {1} "
                         "respectively.".format(tensor1.shape, tensor2.shape))
    if tensor1.shape[dim] != 3:
        raise ValueError("Expected length of input tensors' dim-th ({0}th) dimension to be 3. Got {1} "
                         "instead.".format(dim, tensor1.shape[dim]))


def are_points_close(tensor1: torch.Tensor, tensor2: torch.Tensor, dist_th: Union[float, int],
                     dim: int = -1) -> torch.Tensor:
    """||t1 - t2|| < dist_th along `dim` (fusionutils.py:76-130)."""
    _pair_checks(tensor1, tensor2, dist_th, "dist_th", dim)
    return (tensor1 - tensor2).norm(dim=dim) < dist_th


def are_normals_similar(tensor1: torch.Tensor, tensor2: torch.Tensor, dot_th: Union[float, int],
                        dim: int = -1) -> torch.Tensor:
    """<t1, t2> > dot_th along `dim`; warns if the inputs were not unit length (fusionutils.py:133-195)."""
    _pair_checks(tensor1, tensor2, dot_th, "dot_th", dim)
    dots = (tensor1 * tensor2).sum(dim)
    if dots.numel() > 0 and dots.max() > 1.001:
        warnings.warn("Max of dot product was {0} > 1. Inputs were not normalized along dim ({1}). Was this "
                      "intentional?".format(dots.max(), dim), RuntimeWarning)
    return dots > dot_th


# --------------------------------------------------------------------------------------------- workspaces
class _Workspace:
    """Per (device, stream, B, H, W) scratch of the fusion kernels: frame header, arg-min slots, candidate bins, scan
    state.  gsx_fusion_frame_records re-arms it for every frame; the arg-min slots are kept zero by the merge kernel,
    and K1r clears those a frame abandoned before its merge left behind.  It is keyed by the CUDA stream as well, so
    maps updated concurrently from different streams or threads never share records."""

    _cache = {}
    _lock = threading.Lock()

    def __init__(self, device, B, H, W):
        nbytes = _C.lib().gsx_fusion_workspace_bytes(B, H, W)
        # zeroed once: the arg-min slots are never cleared per frame (a non-zero slot reads as a winning map row), and
        # the statistics start at 0
        self.buf = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        self.shape = (B, H * W)
        self.assoc = None  # K4's per-pixel record for the free-space step (fuse_and_prune), allocated on first use
        self.rec = None  # K4's (c0, alpha) of every merged pixel, for the embedding merge (KE), allocated on first use

    def zeroed_assoc(self):
        """int32 (B, H*W) buffer for K4's assoc_out, zeroed in stream order (K4 writes only merged / appended pixels)."""
        if self.assoc is None:
            self.assoc = torch.zeros(self.shape, dtype=torch.int32, device=self.buf.device)
        else:
            self.assoc.zero_()
        return self.assoc

    def merge_rec(self):
        """float32 (B, H*W, 2) buffer for K4's merge_rec: KE reads only the records of merged pixels, so it is never
        cleared."""
        if self.rec is None:
            self.rec = torch.empty(self.shape + (2,), dtype=torch.float32, device=self.buf.device)
        return self.rec

    @classmethod
    def get(cls, device, B, H, W):
        key = (str(device), torch.cuda.current_stream(device).cuda_stream, B, H, W)
        with cls._lock:
            ws = cls._cache.get(key)
            if ws is None:
                ws = cls(device, B, H, W)
                cls._cache[key] = ws
        return ws


def _check_frame(rgbdimages):
    if not isinstance(rgbdimages, RGBDImages):
        raise TypeError("Expected rgbdimages to be of type gradslam.RGBDImages. Got {0}.".format(type(rgbdimages)))
    if rgbdimages.shape[1] != 1:
        raise ValueError("Expected rgbdimages to have sequence length of 1. Got {0}.".format(rgbdimages.shape[1]))


def _dense(t, name, device):
    """A tensor whose raw pointer goes to a kernel: float32, on `device`, dense."""
    _C.require_cuda(t, name)
    if t.device != device:
        raise ValueError("gradslam_b200: `{}` is on {} but the map lives on {}".format(name, t.device, device))
    return t.contiguous()


def _sigma_value(sigma):
    if torch.is_tensor(sigma):
        if sigma.requires_grad and torch.is_grad_enabled():
            raise ValueError("gradslam_b200: a sigma that requires grad is not supported by the fused map update "
                             "(d/d sigma is only available through fusionutils.get_alpha)")
        return float(sigma.item())
    return float(sigma)


def _map_ptrs(pointclouds, device):
    """(geometry, colours) buffers of a map the kernels may touch: float32 CUDA, dense, on `device`."""
    geo = _dense(pointclouds._geo, "pointclouds (geometry rows)", device)
    col = _dense(pointclouds._col, "pointclouds (colour rows)", device)
    if geo is not pointclouds._geo or col is not pointclouds._col:  # (never for stores this class allocated)
        pointclouds._geo, pointclouds._col = geo, col
    return geo, col


def _launch_frame_records(ws, frames, sigma, device, world=True):
    """K1r: the live frame's records into the workspace (K2 and K4 evaluate the frame values from its depth);
    world=False keeps camera coordinates."""
    B, _, H, W = frames.shape
    P = H * W
    depth, d_bs = _frame_base(_dense_frame(frames.depth_image, "depth_image", device), P)
    K = _dense(frames.intrinsics.detach(), "intrinsics", device)
    poses = _dense(frames.poses.detach(), "poses", device) if (world and frames.poses is not None) else None
    _C.launch("gsx_fusion_frame_records", depth, d_bs, K, 16, poses, 16, B, H, W, sigma, ws.buf)
    # K2 and K4 read this depth (it may be a dense copy made just above): keep it alive until the next frame's records
    # replace it, which is after this frame's merge in stream order
    ws.depth = depth


def _dense_frame(t, name, device):
    """Frame tensors may be views of a (B,L,...) sequence tensor (frame s of every element): the kernels take a base
    pointer plus the element stride, so only the per-frame block has to be dense (see _frame_base)."""
    _C.require_cuda(t, name)
    if t.device != device:
        raise ValueError("gradslam_b200: `{}` is on {} but the map lives on {}".format(name, t.device, device))
    return t


def _embedding_frame(e, device):
    """(B,1,H,W,D) channels-last embedding image ((B,1,h,w,D) when upsampled) -> (base tensor, element stride) for
    KE."""
    if not e.is_cuda or e.device != device:
        raise ValueError("gradslam_b200: `embeddings` is on {} but the map lives on {}".format(e.device, device))
    return _frame_base(e.detach(), e.shape[2] * e.shape[3] * e.shape[4])


def _launch_merge_append(pointclouds, frames, ws, assoc=None, radii=False):
    """K4 on the current workspace state (frame records + per-pixel winners); radii: write surfel radii (slot 7).  A
    frame with embeddings runs K4 with its merge record, then KE on the map's embedding store (the upsampled KE when
    the frame's embedding image is coarser than the depth)."""
    B, _, H, W = frames.shape
    P = H * W
    dev = pointclouds.device
    rgb, c_bs = _frame_base(_dense_frame(frames.rgb_image, "rgb_image", dev), P * 3)
    geo, col = _map_ptrs(pointclouds, dev)
    cin = pointclouds._counts_dev[pointclouds._cur]
    cout = pointclouds._counts_dev[pointclouds._cur ^ 1]
    if frames.embeddings is None:
        _C.launch("gsx_fusion_merge_append_radii", geo, col, 1 if pointclouds._has_cc else 0, cin, cout,
                  pointclouds.capacity, rgb, c_bs, B, H, W, ws.buf, pointclouds._overflow_flag(), assoc,
                  1 if radii else 0)
    else:
        e, e_bs = _embedding_frame(frames.embeddings, dev)
        if pointclouds._emb is None:  # (a map this update starts)
            pointclouds._alloc_embeddings(e.shape[-1], e.dtype)
        emb = pointclouds._emb = pointclouds._emb.contiguous()
        assoc = ws.zeroed_assoc() if assoc is None else assoc
        rec = ws.merge_rec()
        _C.launch("gsx_fusion_merge_append_rec", geo, col, 1 if pointclouds._has_cc else 0, cin, cout,
                  pointclouds.capacity, rgb, c_bs, B, H, W, ws.buf, pointclouds._overflow_flag(), assoc, rec,
                  1 if radii else 0)
        if frames.upsample_embeddings:
            eh, ew = frames.embeddings.shape[2], frames.embeddings.shape[3]
            _C.launch("gsx_embed_merge_append_upsampled", emb, pointclouds.capacity, e, e_bs, assoc, rec, B, H, W, eh,
                      ew, e.shape[-1], EMBED_DTYPES[e.dtype])
        else:
            _C.launch("gsx_embed_merge_append", emb, pointclouds.capacity, e, e_bs, assoc, rec, B, H, W, e.shape[-1],
                      EMBED_DTYPES[e.dtype])
    pointclouds._mark_device_updated(pointclouds._bound + P)


def _prepare_map(pointclouds, frames, with_features):
    """Makes sure the map has storage for B elements with room for one more frame."""
    B, _, H, W = frames.shape
    if not pointclouds.has_points:
        pointclouds.device = frames.device
        pointclouds._allocate(B, 2 * H * W, 1 if with_features else 0)
    elif len(pointclouds) != B:
        raise ValueError("Expected equal batch sizes for pointclouds and rgbdimages. Got {0} and {1} "
                         "respectively.".format(len(pointclouds), B))
    if pointclouds._bound + H * W > pointclouds.capacity:
        pointclouds._host_counts()  # one sync tightens the bound before we decide to grow
    pointclouds.reserve(pointclouds._bound + H * W)


def _append_valid_pixels(pointclouds, frames, global_coordinates=True, sigma=0.6):
    """Stable append of every valid pixel (K4 with no matches): update_map_aggregate / pointclouds_from_rgbdimages."""
    _check_frame(frames)
    frames = frames.to_channels_last()
    _C.require_cuda(frames.depth_image, "depth_image")
    had_points = pointclouds.has_points
    if had_points and not (pointclouds.has_normals and pointclouds.has_colors):
        raise ValueError("Pointclouds must have normals and colors to aggregate frames into it")
    if had_points and pointclouds._feat is not None:
        raise ValueError("pointclouds to append and to be appended must have the same number of features")
    with_features = pointclouds.has_features if had_points else False
    _check_embeddings(pointclouds, frames)
    _prepare_map(pointclouds, frames, with_features)
    B, _, H, W = frames.shape
    dev = pointclouds.device
    ws = _Workspace.get(dev, B, H, W)
    _launch_frame_records(ws, frames, _sigma_value(sigma), dev, world=global_coordinates)
    _launch_merge_append(pointclouds, frames, ws)
    return pointclouds


def _check_embeddings(pointclouds, rgbdimages):
    """A map update carries embeddings when the map and the frame both have them, or the map is empty and the frame has
    them; any other mismatch is refused, as is half precision in the differentiable mode.  Host-side only."""
    e = rgbdimages.embeddings
    if pointclouds.has_points:
        if pointclouds.has_embeddings != (e is not None):
            raise ValueError("the map {} embeddings but the frame {}: both or neither must carry them".format(
                "has" if pointclouds.has_embeddings else "has no", "does not" if e is None else "does"))
        if e is not None:
            D = e.shape[rgbdimages.cdim]
            if (pointclouds._emb.shape[2], pointclouds._emb.dtype) != (D, e.dtype):
                raise ValueError("the map's embeddings (D={}, {}) and the frame's (D={}, {}) differ".format(
                    pointclouds._emb.shape[2], pointclouds._emb.dtype, D, e.dtype))
    if e is not None and e.dtype != torch.float32 and _wants_grad(pointclouds, rgbdimages):
        raise TypeError("the differentiable map update supports float32 embeddings only; got {}".format(e.dtype))


def _refuse_embeddings(pointclouds, what, rgbdimages=None):
    if (pointclouds.has_points and pointclouds.has_embeddings) or (rgbdimages is not None and
                                                                   rgbdimages.embeddings is not None):
        raise ValueError("{} is not supported on maps with embeddings: its compaction would have to move the "
                         "embedding rows too".format(what))


def _check_fusion_inputs(pointclouds, rgbdimages):
    """A fused update needs the live frame's poses and a map with normals, colours and one confidence count per point."""
    if rgbdimages.poses is None:
        raise ValueError("rgbdimages must have poses for map fusion")
    if pointclouds.has_points:
        for what in ("normals", "colors", "features"):
            if not getattr(pointclouds, "has_" + what):
                raise ValueError("Pointclouds must have {} for map fusion, but did not.".format(what))
        if pointclouds.num_features != 1:
            raise ValueError("Pointclouds features must be a single confidence count per point for map fusion.")


def _update_in_place(pointclouds, frames, sigma, dist_th=None, dot_th=None, table=None, assoc_out=None, radii=False):
    """K1r, the association (K2 with dist_th / dot_th, or the rows of `table`), then K4, in place.  assoc_out: a list
    that receives K4's per-pixel record (B, H*W) int32; radii: K4 writes surfel radii."""
    frames = frames.to_channels_last()
    _C.require_cuda(frames.depth_image, "depth_image")
    B, _, H, W = frames.shape
    _prepare_map(pointclouds, frames, True)
    dev = pointclouds.device
    ws = _Workspace.get(dev, B, H, W)
    _launch_frame_records(ws, frames, _sigma_value(sigma), dev)
    _launch_association(ws, pointclouds, frames, dist_th=dist_th, dot_th=dot_th, table=table)
    assoc = None
    if assoc_out is not None:
        assoc = ws.zeroed_assoc()
        assoc_out.append(assoc)
    _launch_merge_append(pointclouds, frames, ws, assoc, radii)
    return pointclouds


def _check_surfel_radii(surfel_radii):
    if not isinstance(surfel_radii, bool):
        raise TypeError("surfel_radii must be of type bool; but was of type {}.".format(type(surfel_radii)))


# --------------------------------------------------------------------------------------------- table API
def _compact(flags: torch.Tensor) -> torch.Tensor:
    """Ascending indices of the non-zero entries of a flat uint8 CUDA tensor (stable compaction kernel)."""
    n = flags.numel()
    dev = flags.device
    scratch = torch.zeros(_C.lib().gsx_compact_scratch_bytes(n), dtype=torch.uint8, device=dev)
    idx = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    _C.launch("gsx_compact_indices", flags, n, idx, cnt, scratch, 1)
    return idx[: int(cnt.item())]  # the table's length is data dependent: this is the API's one host sync


def _check_table(pc2im_bnhw):
    if not torch.is_tensor(pc2im_bnhw):
        raise TypeError("Expected input pc2im_bnhw to be of type torch.Tensor. Got {0} instead.".format(
            type(pc2im_bnhw)))
    if pc2im_bnhw.dtype != torch.int64:
        raise TypeError("Expected input pc2im_bnhw to have dtype of torch.int64 (torch.long), not {0}.".format(
            pc2im_bnhw.dtype))


def _check_table_shape(pc2im_bnhw):
    if pc2im_bnhw.ndim != 2:
        raise ValueError("Expected pc2im_bnhw.ndim of 2. Got {0}.".format(pc2im_bnhw.ndim))
    if pc2im_bnhw.shape[1] != 4:
        raise ValueError("Expected pc2im_bnhw.shape[1] to be 4. Got {0}.".format(pc2im_bnhw.shape[1]))


def _check_pc(pointclouds):
    if not isinstance(pointclouds, Pointclouds):
        raise TypeError("Expected pointclouds to be of type gradslam.Pointclouds. Got {0}.".format(type(pointclouds)))


def _check_batch(pointclouds, rgbdimages):
    if len(rgbdimages) != len(pointclouds):
        raise ValueError("Expected equal batch sizes for pointclouds and rgbdimages. Got {0} and {1} "
                         "respectively.".format(len(pointclouds), len(rgbdimages)))


def find_active_map_points(pointclouds: Pointclouds, rgbdimages: RGBDImages) -> torch.Tensor:
    """int64 (A,4) rows [b, n, h, w] of the map points that project inside the live frame, in (b, n) order
    (fusionutils.py:198-287)."""
    _check_pc(pointclouds)
    _check_frame(rgbdimages)
    device = pointclouds.device
    if not pointclouds.has_points:
        return torch.empty((0, 4), dtype=torch.int64, device=device)
    _check_batch(pointclouds, rgbdimages)
    frames = rgbdimages.to_channels_last()
    B, _, H, W = frames.shape
    geo = _dense(pointclouds._geo, "pointclouds (geometry rows)", device)
    width = min(max(pointclouds._bound, 1), pointclouds.capacity)
    flags = torch.empty((B, width), dtype=torch.uint8, device=device)
    hw = torch.empty((B, width), dtype=torch.int32, device=device)
    poses, K = _dense(frames.poses, "poses", device), _dense(frames.intrinsics, "intrinsics", device)
    _C.launch("gsx_active_eval", geo, pointclouds._counts_dev[pointclouds._cur], pointclouds.capacity, width, poses, 16,
              K, 16, B, H, W, flags, hw)
    idx = _compact(flags.view(-1))
    pix = hw.view(-1)[idx].to(torch.int64)
    table = torch.stack([idx // width, idx % width, pix // W, pix % W], dim=1)
    if table.shape[0] == 0:
        warnings.warn("No active map points were found")
    return table


def find_similar_map_points(pointclouds: Pointclouds, rgbdimages: RGBDImages, pc2im_bnhw: torch.Tensor,
                            dist_th: Union[float, int], dot_th: Union[float, int]):
    """Rows of the active table whose map point is close to, and has a normal similar to, the frame point of the
    pixel it lands on.  Returns (int64 (S,4), bool (A,)) (fusionutils.py:290-411)."""
    _check_pc(pointclouds)
    if not isinstance(rgbdimages, RGBDImages):
        raise TypeError("Expected rgbdimages to be of type gradslam.RGBDImages. Got {0}.".format(type(rgbdimages)))
    _check_table(pc2im_bnhw)
    if rgbdimages.shape[1] != 1:
        raise ValueError("Expected rgbdimages to have sequence length of 1. Got {0}.".format(rgbdimages.shape[1]))
    _check_table_shape(pc2im_bnhw)
    device = pointclouds.device
    if not pointclouds.has_points or pc2im_bnhw.shape[0] == 0:
        return torch.empty((0, 4), dtype=torch.int64, device=device), torch.empty(0, dtype=torch.bool, device=device)
    _check_batch(pointclouds, rgbdimages)
    if not pointclouds.has_normals:
        raise ValueError("Pointclouds must have normals for finding similar map points, but did not.")
    frames = rgbdimages.to_channels_last()
    B, _, H, W = frames.shape
    table = pc2im_bnhw.contiguous()
    rows = table.shape[0]
    gv, gn = frames.global_vertex_map.contiguous(), frames.global_normal_map.contiguous()
    geo = _dense(pointclouds._geo, "pointclouds (geometry rows)", device)
    flags = torch.empty(rows, dtype=torch.uint8, device=device)
    _C.launch("gsx_similar_eval", table, rows, geo, pointclouds.capacity, gv, gn, B, H, W, float(dist_th), float(dot_th),
              flags)
    keep = _compact(flags)
    similar = table[keep]
    if similar.shape[0] == 0:
        warnings.warn("No similar map points were found (despite total {0} active points across the batch)".format(
            rows), RuntimeWarning)
    return similar, flags.bool()


def find_best_unique_correspondences(pointclouds: Pointclouds, rgbdimages: RGBDImages,
                                     pc2im_bnhw: torch.Tensor) -> torch.Tensor:
    """One row per live pixel: among the candidates of a pixel keep the largest confidence count, then the
    smallest ray distance, then the smallest index.  Output sorted by (b, h, w) (fusionutils.py:414-546); the
    reference's torch.unique(dim=0) row sort becomes a per-pixel atomic arg-min."""
    _check_pc(pointclouds)
    _check_table(pc2im_bnhw)
    if rgbdimages.shape[1] != 1:
        raise ValueError("Expected rgbdimages to have sequence length of 1. Got {0}.".format(rgbdimages.shape[1]))
    _check_table_shape(pc2im_bnhw)
    device = pointclouds.device
    if not pointclouds.has_points or pc2im_bnhw.shape[0] == 0:
        return torch.empty((0, 4), dtype=torch.int64, device=device)
    _check_batch(pointclouds, rgbdimages)
    if not pointclouds.has_features:
        raise ValueError("Pointclouds must have features for finding best unique correspondences, but did not.")
    frames = rgbdimages.to_channels_last()
    B, _, H, W = frames.shape
    table = pc2im_bnhw.contiguous()
    if pointclouds.num_features != 1:
        raise ValueError("Pointclouds features must be a single confidence count per point.")
    gv = frames.global_vertex_map.contiguous()
    geo = _dense(pointclouds._geo, "pointclouds (geometry rows)", device)
    records = torch.empty(B * H * W, dtype=torch.int32, device=device)  # 4-byte arg-min slots (scratch)
    pflags = torch.empty(B * H * W, dtype=torch.uint8, device=device)
    pn = torch.empty(B * H * W, dtype=torch.int64, device=device)
    _C.launch("gsx_unique_select", table, table.shape[0], geo, pointclouds.capacity, gv, B, H, W, records, pflags, pn)
    pix = _compact(pflags)
    rem = pix % (H * W)
    return torch.stack([pix // (H * W), pn[pix], rem // W, rem % W], dim=1)


def find_correspondences(pointclouds: Pointclouds, rgbdimages: RGBDImages, dist_th: Union[float, int],
                         dot_th: Union[float, int]) -> torch.Tensor:
    """active -> similar -> best unique (fusionutils.py:549-577)."""
    pc2im_bnhw = find_active_map_points(pointclouds, rgbdimages)
    pc2im_bnhw, _ = find_similar_map_points(pointclouds, rgbdimages, pc2im_bnhw, dist_th, dot_th)
    return find_best_unique_correspondences(pointclouds, rgbdimages, pc2im_bnhw)


def fuse_with_map(pointclouds: Pointclouds, rgbdimages: RGBDImages, pc2im_bnhw: torch.Tensor,
                  sigma: Union[torch.Tensor, float, int], inplace: bool = False, *,
                  surfel_radii: bool = False) -> Pointclouds:
    """Merges the corresponding points of `pc2im_bnhw` (unique rows) and appends the unmatched valid pixels
    (fusionutils.py:580-722).  surfel_radii (extension): as in update_map_fusion."""
    _check_pc(pointclouds)
    _check_surfel_radii(surfel_radii)
    if not isinstance(rgbdimages, RGBDImages):
        raise TypeError("Expected rgbdimages to be of type gradslam.RGBDImages. Got {0}.".format(type(rgbdimages)))
    _check_table(pc2im_bnhw)
    _check_table_shape(pc2im_bnhw)
    if pointclouds.has_points:
        for what in ("normals", "colors"):
            if not getattr(pointclouds, "has_" + what):
                raise ValueError("Pointclouds must have {} for map fusion, but did not.".format(what))
        if not pointclouds.has_features:
            raise ValueError("Pointclouds must have features (ccounts) for map fusion, but did not.")
    _check_frame(rgbdimages)
    _check_embeddings(pointclouds, rgbdimages)
    if not inplace:
        pointclouds = pointclouds.clone()
    return _fuse(pointclouds, rgbdimages, sigma, table=pc2im_bnhw, radii=surfel_radii)


def _launch_association(ws, pointclouds, frames, dist_th=None, dot_th=None, table=None):
    """The per-pixel winners K4 merges into, after K1r: the rows of a unique correspondence `table`, or K2 over the
    map's rows with dist_th / dot_th (neither: no winners, every valid pixel is appended).  Index-only: no gradient flows
    through the association (fusionutils.py:523)."""
    if pointclouds._bound == 0:
        return
    B, _, H, W = frames.shape
    dev = pointclouds.device
    if table is not None:
        if table.shape[0] != 0:
            table = table.to(dev).contiguous()
            _C.launch("gsx_records_from_table", table, table.shape[0], pointclouds.capacity, B, H, W, ws.buf)
    elif dist_th is not None:
        geo = _dense(pointclouds._geo.detach(), "pointclouds (geometry rows)", dev)
        poses = _dense(frames.poses.detach(), "poses", dev)
        K = _dense(frames.intrinsics.detach(), "intrinsics", dev)
        _C.launch("gsx_fusion_project_select", geo, pointclouds._counts_dev[pointclouds._cur], pointclouds.capacity,
                  pointclouds._bound, poses, 16, K, 16, B, H, W, float(dist_th), float(dot_th), ws.buf)


# --------------------------------------------------------------------------------------------- differentiable mode
def _wants_grad(pointclouds, frames):
    if not torch.is_grad_enabled():
        return False
    ts = [frames.depth_image, frames.poses, frames.rgb_image, frames.intrinsics, frames.embeddings,
          pointclouds._emb] + pointclouds._grad_tensors()
    return any(torch.is_tensor(t) and t.requires_grad for t in ts)


class _MergeAppendFn(torch.autograd.Function):
    """K4 as one differentiable op: (pre-merge map rows, frame maps) -> updated map rows.  forward =
    gsx_fusion_merge_append_radii (surfel radii on or off) on a copy of the map (also records where every pixel went),
    backward = gsx_fusion_merge_append_bwd; both hand-written kernels, both on the packed row layout (the public
    points / normals / colors / features / radii tensors are slices of the rows, so autograd carries the gradients in
    and out of the rows by itself).  The radii carry no gradient: the gradient w.r.t. `radii_padded` is identically
    zero.  The frame records and the per-pixel winners must already sit in the fusion workspace
    (K1r; K2, or gsx_records_from_table); the winners are index-only, as in the reference (fusionutils.py:523).
    With the map's embeddings `emb` (B, cap, D) and the frame's `e` (B, 1, H, W, D), float32, K4 also records each
    merge's weights and KE (gsx_embed_merge_append) merges the embeddings, a third output; the backward runs
    gsx_embed_merge_bwd first and hands its d c0 / d alpha terms to K4's (gsx_fusion_merge_append_bwd_emb).  A frame
    with upsample_embeddings carries its coarse (B, 1, h, w, D) image instead, through the _upsampled entry points,
    and gets its gradient in that shape."""

    @staticmethod
    def forward(ctx, pack, geo, col, gv, gn, rgb, vloc, emb=None, e=None):
        pointclouds, frames, sigma, ws, _, radii = pack
        B, _, H, W = frames.shape
        P = H * W
        dev = geo.device
        bound, cap_in, cap_out = pointclouds._bound, geo.shape[1], pointclouds._bound + P
        outs = []
        for t in (geo, col):
            o = torch.zeros((B, cap_out, t.shape[2]), dtype=torch.float32, device=dev)
            if bound > 0:
                o[:, :bound] = t.detach()[:, :bound]
            outs.append(o)
        gv_c, gn_c, rgb_c, vloc_c = (t.detach().contiguous() for t in (gv, gn, rgb, vloc))
        counts_in = pointclouds._counts_dev[pointclouds._cur].clone()
        counts_out = pointclouds._counts_dev[pointclouds._cur ^ 1]
        assoc = torch.zeros((B, P), dtype=torch.int32, device=dev)
        with_cc = 1 if pointclouds._has_cc else 0
        ctx.emb = None
        if e is None:
            _C.launch("gsx_fusion_merge_append_radii", outs[0], outs[1], with_cc, counts_in, counts_out, cap_out, rgb_c,
                      P * 3, B, H, W, ws.buf, pointclouds._overflow_flag(), assoc, 1 if radii else 0)
        else:
            D = e.shape[-1]
            emb_out = torch.zeros((B, cap_out, D), dtype=torch.float32, device=dev)
            if bound > 0:
                emb_out[:, :bound] = emb.detach()[:, :bound]
            rec = torch.empty((B, P, 2), dtype=torch.float32, device=dev)
            e_c = e.detach().contiguous()
            _C.launch("gsx_fusion_merge_append_rec", outs[0], outs[1], with_cc, counts_in, counts_out, cap_out, rgb_c,
                      P * 3, B, H, W, ws.buf, pointclouds._overflow_flag(), assoc, rec, 1 if radii else 0)
            up = (e.shape[2], e.shape[3]) if frames.upsample_embeddings else None  # the coarse image's (h, w)
            if up is None:
                _C.launch("gsx_embed_merge_append", emb_out, cap_out, e_c, P * D, assoc, rec, B, H, W, D, 0)
            else:
                _C.launch("gsx_embed_merge_append_upsampled", emb_out, cap_out, e_c, up[0] * up[1] * D, assoc, rec, B,
                          H, W, up[0], up[1], D, 0)
            outs.append(emb_out)
            ctx.emb = (rec, emb.detach().contiguous(), e_c, e.shape, up)
        if pack[4] is not None:  # (fuse_and_prune's free-space step reads it)
            pack[4].append(assoc)
        ctx.saved = (assoc, counts_in, geo.detach(), col.detach(), gv_c, gn_c, rgb_c, vloc_c)
        ctx.dims = (B, H, W, cap_in, cap_out, float(sigma), with_cc)
        ctx.shapes = (gv.shape, rgb.shape)
        return tuple(outs)

    @staticmethod
    def backward(ctx, g_geo, g_col, g_emb=None):
        assoc, counts_in, geo, col, gv, gn, rgb, vloc = ctx.saved
        B, H, W, cap_in, cap_out, sigma, with_cc = ctx.dims
        dev = assoc.device
        gs = [None if g is None else g.contiguous().float() for g in (g_geo, g_col)]
        geo_c, col_c = geo.contiguous(), col.contiguous()
        d_map = [torch.empty_like(geo_c), torch.empty_like(col_c)]
        d_frame = [torch.empty((B, 1, H, W, 3), dtype=torch.float32, device=dev) for _ in range(4)]
        gv_shape, rgb_shape = ctx.shapes
        if ctx.emb is None:
            _C.launch("gsx_fusion_merge_append_bwd", assoc, counts_in, geo_c, col_c, with_cc, cap_in, *gs, cap_out, gv,
                      gn, rgb, vloc, B, H, W, sigma, *d_map, *d_frame)
            return (None, d_map[0], d_map[1], d_frame[0].view(gv_shape), d_frame[1].view(gv_shape),
                    d_frame[2].view(rgb_shape), d_frame[3].view(gv_shape))
        rec, emb, e, e_shape, up = ctx.emb
        D = e.shape[-1]
        d_emb = torch.empty_like(emb)
        d_e = torch.empty_like(e)
        d_w = torch.empty((2, B, H * W), dtype=torch.float32, device=dev)  # d c0, d alpha per pixel
        g_emb = None if g_emb is None else g_emb.contiguous()
        if up is None:
            _C.launch("gsx_embed_merge_bwd", assoc, rec, counts_in, emb, cap_in, e, g_emb, cap_out, B, H, W, D, d_emb,
                      d_e, d_w[0], d_w[1])
        else:
            _C.launch("gsx_embed_merge_bwd_upsampled", assoc, rec, counts_in, emb, cap_in, e, g_emb, cap_out, B, H, W,
                      up[0], up[1], D, d_emb, d_e, d_w[0], d_w[1])
        _C.launch("gsx_fusion_merge_append_bwd_emb", assoc, counts_in, geo_c, col_c, with_cc, cap_in, *gs, cap_out, gv,
                  gn, rgb, vloc, B, H, W, sigma, d_w[0], d_w[1], *d_map, *d_frame)
        return (None, d_map[0], d_map[1], d_frame[0].view(gv_shape), d_frame[1].view(gv_shape),
                d_frame[2].view(rgb_shape), d_frame[3].view(gv_shape), d_emb, d_e.view(e_shape))


def _update_differentiable(pointclouds, frames, sigma, with_features, dist_th=None, dot_th=None, table=None,
                           assoc_out=None, radii=False):
    """Map update when a gradient is requested: K1 (differentiable op, for the backward) -> frame records ->
    association (K2 kernel, or the rows of `table`; index-only) -> K4 (differentiable op), out of place so the pre-merge
    map survives for the backward.  K4's forward re-evaluates the frame values from depth, as the in-place path does,
    and K1's maps equal them bit for bit.  assoc_out: a list that receives K4's per-pixel record."""
    frames = frames.to_channels_last()
    _C.require_cuda(frames.depth_image, "depth_image")
    B, _, H, W = frames.shape
    P = H * W
    if not pointclouds.has_points:
        pointclouds.device = frames.device
        pointclouds._allocate(B, 1, 1 if with_features else 0)
    elif len(pointclouds) != B:
        raise ValueError("Expected equal batch sizes for pointclouds and rgbdimages. Got {0} and {1} "
                         "respectively.".format(len(pointclouds), B))
    dev = pointclouds.device
    e = frames.embeddings
    emb_args = ()
    if e is not None:
        if pointclouds._emb is None:
            pointclouds._alloc_embeddings(e.shape[-1], e.dtype)
        _embedding_frame(e, dev)  # (device check)
        emb_args = (pointclouds._emb, e)
    sig = _sigma_value(sigma)
    gv, gn, vloc = frames.global_vertex_map, frames.global_normal_map, frames.vertex_map  # K1, carries its backward
    ws = _Workspace.get(dev, B, H, W)
    _launch_frame_records(ws, frames, sig, dev)
    _launch_association(ws, pointclouds, frames, dist_th=dist_th, dot_th=dot_th, table=table)
    outs = _MergeAppendFn.apply((pointclouds, frames, sig, ws, assoc_out, radii), pointclouds._geo, pointclouds._col,
                                gv, gn, frames.rgb_image, vloc, *emb_args)
    pointclouds._geo, pointclouds._col = outs[0], outs[1]
    if e is not None:
        pointclouds._emb = outs[2]
    pointclouds._uninit = False
    pointclouds._mark_device_updated(pointclouds._bound + P)
    return pointclouds


def _fuse(pointclouds, frames, sigma, dist_th=None, dot_th=None, table=None, assoc_out=None, radii=False):
    """The fused map update: the differentiable op chain when a gradient is requested, else in place.  A frame without
    poses (only fuse_with_map accepts one) has no world-frame maps for the differentiable chain and is fused in place."""
    if _wants_grad(pointclouds, frames) and frames.poses is not None:
        return _update_differentiable(pointclouds, frames, sigma, True, dist_th, dot_th, table, assoc_out, radii)
    return _update_in_place(pointclouds, frames, sigma, dist_th, dot_th, table, assoc_out, radii)


# --------------------------------------------------------------------------------------------- unstable surfels
def _check_history(pointclouds, t_max):
    """Raises before anything is launched if the map was pruned with another max_unstable_age."""
    h = pointclouds._prune
    if h is not None and h.t_max != t_max:
        raise ValueError("max_unstable_age ({}) differs from the one this map was pruned with ({})".format(
            t_max, h.t_max))


def _prune_scratch(B, capacity, device):
    return torch.empty(_C.lib().gsx_fusion_prune_scratch_bytes(B, capacity), dtype=torch.uint8, device=device)


class _PruneFn(torch.autograd.Function):
    """The prune as one differentiable op on the packed rows: forward = `prune` (a gsx_fusion_prune launch) on a copy of
    the rows, recording where every row went (keep_map); backward = gsx_fusion_prune_bwd, a gather.  The removal itself
    is a decision on the confidence and the geometry and carries no gradient, as an index_select would not."""

    @staticmethod
    def forward(ctx, prune, counts, geo, col):
        B, cap = geo.shape[0], geo.shape[1]
        geo_o, col_o = geo.detach().clone(), col.detach().clone()
        keep_map = torch.arange(cap, dtype=torch.int32, device=geo.device).repeat(B, 1)  # rows before the scan: identity
        ctx.saved = (keep_map, counts.clone())
        prune(geo_o, col_o, keep_map)
        return geo_o, col_o

    @staticmethod
    def backward(ctx, g_geo, g_col):
        keep_map, counts_in = ctx.saved
        B, cap = keep_map.shape
        gs = [None if g is None else g.contiguous().float() for g in (g_geo, g_col)]
        d_geo = torch.empty((B, cap, 8), dtype=torch.float32, device=keep_map.device)
        d_col = torch.empty((B, cap, 4), dtype=torch.float32, device=keep_map.device)
        _C.launch("gsx_fusion_prune_bwd", keep_map, counts_in, cap, gs[0], gs[1], cap, B, d_geo, d_col)
        return None, None, d_geo, d_col


class _PruneMergeFn(torch.autograd.Function):
    """_PruneFn with merging of overlapping surfels: the forward also records every absorbed pair and keeps the pairs'
    pre-step rows (b, m, n and rows m, n: 104 bytes per pair, about 1 % of the map's rows at 640x480), and the backward
    (gsx_fusion_prune_merge_bwd) adds the quotient rule of each absorption to the gather.  Finding the pairs costs one
    host synchronisation per pruned step (their number sizes the record)."""

    @staticmethod
    def forward(ctx, prune, counts, geo, col):
        B, cap = geo.shape[0], geo.shape[1]
        geo_o, col_o = geo.detach().clone(), col.detach().clone()
        keep_map = torch.arange(cap, dtype=torch.int32, device=geo.device).repeat(B, 1)  # rows before the scan: identity
        absorbed = torch.full((B, cap), -1, dtype=torch.int32, device=geo.device)
        counts_in = counts.clone()
        prune(geo_o, col_o, keep_map, absorbed)
        bm = torch.nonzero(absorbed >= 0)
        b, m = bm[:, 0], bm[:, 1]
        n = absorbed[b, m].long()
        rows = torch.stack([m, n], 1)
        pair_geo = geo.detach()[b.unsqueeze(1), rows].contiguous()  # (A, 2, 8)
        pair_col = col.detach()[b.unsqueeze(1), rows].contiguous()  # (A, 2, 4)
        pairs = torch.stack([b, m, n], 1).to(torch.int32).contiguous()
        ctx.saved = (keep_map, counts_in, pairs, pair_geo, pair_col)
        return geo_o, col_o

    @staticmethod
    def backward(ctx, g_geo, g_col):
        keep_map, counts_in, pairs, pair_geo, pair_col = ctx.saved
        B, cap = keep_map.shape
        gs = [None if g is None else g.contiguous().float() for g in (g_geo, g_col)]
        d_geo = torch.empty((B, cap, 8), dtype=torch.float32, device=keep_map.device)
        d_col = torch.empty((B, cap, 4), dtype=torch.float32, device=keep_map.device)
        _C.launch("gsx_fusion_prune_merge_bwd", keep_map, counts_in, cap, pairs, pair_geo, pair_col, pairs.shape[0],
                  gs[0], gs[1], cap, B, d_geo, d_col)
        return None, None, d_geo, d_col


def _prune(pointclouds, stable_confidence, t_max, free_space=None, merge_dot_th=None):
    """One pruned step of the map, in place: the age rule and, with free_space = (assoc, K, poses, H, W, margin) of the
    step's K4, the free-space rule, and with merge_dot_th as well, merging of overlapping surfels.  A differentiable op
    when the map's rows require grad.  The map's pruning history is created at its first pruned step (rows already in
    the map count as created then)."""
    h = pointclouds._prune
    if h is None:
        h = pointclouds._prune = _PruneHistory.fresh(len(pointclouds), t_max, pointclouds.device)
    B, cap, dev = len(pointclouds), pointclouds.capacity, pointclouds.device
    counts = pointclouds._counts_dev[pointclouds._cur]
    scratch = _prune_scratch(B, cap, dev)
    fs = (None, None, 0, None, 0, 0, 0, 0.0, None, 0)  # the age rule alone
    if free_space is not None:
        assoc, K, poses, H, W, margin = free_space
        fs_scratch = torch.empty(_C.lib().gsx_fusion_free_space_scratch_bytes(B, H, W, cap), dtype=torch.uint8,
                                 device=dev)
        fs = (assoc, K, 16, poses, 16, H, W, float(margin), fs_scratch, fs_scratch.numel())

    if merge_dot_th is None:
        def launch(geo, col, keep_map):
            _C.launch("gsx_fusion_prune", geo, col, counts, cap, h.ring, h.t_max + 2, h.step, h.t_max,
                      float(stable_confidence), B, keep_map, scratch, scratch.numel(), *fs)
        fn = _PruneFn
    else:
        ms = torch.empty(_C.lib().gsx_fusion_merge_scratch_bytes(B, H, W, cap), dtype=torch.uint8, device=dev)

        def launch(geo, col, keep_map, absorbed=None):
            _C.launch("gsx_fusion_prune_merge", geo, col, counts, cap, h.ring, h.t_max + 2, h.step, h.t_max,
                      float(stable_confidence), B, keep_map, scratch, scratch.numel(), *fs, float(merge_dot_th), ms,
                      ms.numel(), absorbed)
        fn = _PruneMergeFn

    if torch.is_grad_enabled() and any(t.requires_grad for t in pointclouds._grad_tensors()):
        pointclouds._geo, pointclouds._col = fn.apply(launch, counts, pointclouds._geo, pointclouds._col)
    else:
        launch(*_map_ptrs(pointclouds, dev), None)
    # one more pruned step; the sizes changed on the device (the host bound stays an upper bound), and rows past the new
    # sizes hold stale values until a padded view zeroes them
    h.step += 1
    pointclouds._counts_host = None
    pointclouds._list_cache = {}
    pointclouds._uninit = pointclouds._tail_dirty = True


def prune_unstable(pointclouds: Pointclouds, stable_confidence: float, max_unstable_age: int) -> Pointclouds:
    """Removes unstable surfels, in place, as one pruned step of the map (Keller et al. 2013, section 4.3; an extension:
    gradslam keeps every surfel).  The rows created `max_unstable_age` pruned steps ago whose confidence (the
    `features_padded` value: gradslam's alpha summed over merges) is still below `stable_confidence` are removed; every
    other row keeps its order.  Run it after each fused update (PointFusion does, when configured)."""
    _refuse_embeddings(pointclouds, "prune_unstable")
    if not pointclouds.has_points:
        return pointclouds
    if not pointclouds._has_cc or pointclouds._col is None:
        raise ValueError("pruning needs maps with colours and a confidence count per point")
    _check_history(pointclouds, int(max_unstable_age))
    _prune(pointclouds, stable_confidence, int(max_unstable_age))
    return pointclouds


# --------------------------------------------------------------------------------------------- free-space violations
def _check_free_space_margin(margin):
    """free_space_margin: a number (not a bool), >= 0 (inf allowed), not NaN."""
    if isinstance(margin, bool) or not isinstance(margin, (float, int)):
        raise TypeError("free_space_margin must be of type float or int; but was of type {}.".format(type(margin)))
    if math.isnan(margin) or margin < 0:
        raise ValueError("free_space_margin ({}) must be >= 0".format(margin))


def _check_merge_overlapping(merge_overlapping, surfel_radii):
    if not isinstance(merge_overlapping, bool):
        raise TypeError("merge_overlapping must be of type bool; but was of type {}.".format(type(merge_overlapping)))
    if merge_overlapping and not surfel_radii:
        raise ValueError("merge_overlapping needs surfel_radii=True (it merges surfels whose disks overlap)")


def fuse_and_prune(pointclouds: Pointclouds, rgbdimages: RGBDImages, dist_th: Union[float, int],
                   dot_th: Union[float, int], sigma: Union[torch.Tensor, float, int],
                   stable_confidence: Union[float, int], max_unstable_age: int,
                   free_space_margin: Union[float, int], inplace: bool = False, *,
                   surfel_radii: bool = False, merge_overlapping: bool = False) -> Pointclouds:
    """update_map_fusion followed by one pruned step with both of Keller et al.'s (2013, section 4.3) outlier rules
    (an extension: gradslam keeps every surfel).  The age rule is prune_unstable's.  The free-space rule: wherever the
    live frame merged a pixel into a surfel that is stable after the merge (confidence >= stable_confidence), every
    surfel that projects to that same pixel more than `free_space_margin` (metres, camera z) in front of it is removed,
    stable or not.  Unlike the paper (a 4x4-supersampled index map), "in front" is decided at image resolution, at the
    pixel the association's own projection gives.  Both removals are one stable compaction: kept rows keep their order.
    free_space_margin = inf removes no violator (the result is update_map_fusion + prune_unstable).  surfel_radii: as in
    update_map_fusion; the pruning moves whole rows, radius included.

    merge_overlapping (extension, default False; needs surfel_radii=True): in the same step, Keller et al.'s third rule,
    "merge surfels with similar position and normal and overlapping radii".  At every pixel the live frame merged into
    a surfel m that is stable after the merge (and that the free-space rule keeps), the other surfels projecting to that
    pixel are candidates when no pixel merged into them, neither rule removes them, both radii are positive, the normals'
    dot product exceeds dot_th and the disks overlap (centre distance <= r_m + r_n).  The closest candidate (ties: the
    lower index) is absorbed: m becomes the confidence-weighted mean of both surfels (position, normal, colour, radius;
    the confidences add up) and the candidate is removed.  As the free-space rule, this works at the merged pixel, at
    image resolution, not on the paper's 4x4-supersampled index map.  Merging runs with free_space_margin = inf as
    well, which removes no violator.  Gradients flow through the absorption's weighted mean."""
    if not isinstance(pointclouds, Pointclouds):
        raise TypeError("Expected pointclouds to be of type gradslam.Pointclouds. Got {0}.".format(type(pointclouds)))
    _check_frame(rgbdimages)
    _refuse_embeddings(pointclouds, "fuse_and_prune", rgbdimages)
    _check_surfel_radii(surfel_radii)
    _check_merge_overlapping(merge_overlapping, surfel_radii)
    _check_free_space_margin(free_space_margin)
    t_max = int(max_unstable_age)
    _check_history(pointclouds, t_max)
    if pointclouds.has_points and not pointclouds._has_cc:
        raise ValueError("pruning needs maps with colours and a confidence count per point")
    _check_fusion_inputs(pointclouds, rgbdimages)
    if not inplace:
        pointclouds = pointclouds.clone()
    got = []
    _fuse(pointclouds, rgbdimages, sigma, dist_th, dot_th, assoc_out=got, radii=surfel_radii)
    frames = rgbdimages.to_channels_last()
    _, _, H, W = frames.shape
    dev = pointclouds.device
    free_space = (got[0], _dense(frames.intrinsics.detach(), "intrinsics", dev),
                  _dense(frames.poses.detach(), "poses", dev), H, W, free_space_margin)
    _prune(pointclouds, stable_confidence, t_max, free_space, dot_th if merge_overlapping else None)
    return pointclouds


# --------------------------------------------------------------------------------------------- public ops
def update_map_aggregate(pointclouds: Pointclouds, rgbdimages: RGBDImages, inplace: bool = False) -> Pointclouds:
    """Appends every valid live-frame pixel to the maps (fusionutils.py:725-758)."""
    if not isinstance(pointclouds, Pointclouds):
        raise TypeError("Expected pointclouds to be of type gradslam.Pointclouds. Got {0}.".format(type(pointclouds)))
    if not isinstance(rgbdimages, RGBDImages):
        raise TypeError("Expected rgbdimages to be of type gradslam.RGBDImages. Got {0}.".format(type(rgbdimages)))
    if pointclouds.has_points and pointclouds.has_features:
        # the reference appends a features-less cloud built from the frame (structures/utils.py:7-57) and
        # Pointclouds.append_points refuses the mismatch (pointclouds.py:1170-1177)
        raise ValueError("pointclouds to append and to be appended must either both have or not have features: "
                         "(False != True)")
    _check_embeddings(pointclouds, rgbdimages)
    if not inplace:
        pointclouds = pointclouds.clone()
    if _wants_grad(pointclouds, rgbdimages):
        _check_frame(rgbdimages)
        return _update_differentiable(pointclouds, rgbdimages, 0.6, False)
    return _append_valid_pixels(pointclouds, rgbdimages, True)


def update_map_fusion(pointclouds: Pointclouds, rgbdimages: RGBDImages, dist_th: Union[float, int],
                      dot_th: Union[float, int], sigma: Union[torch.Tensor, float, int],
                      inplace: bool = False, *, surfel_radii: bool = False) -> Pointclouds:
    """PointFusion update of the maps with one live frame (fusionutils.py:761-789).

    surfel_radii (extension, default False): every merged or appended surfel also gets a radius, readable as
    `radii_padded` / `radii_list`: min(2 r0, r0 / |n_z|) with r0 = sqrt(2) d / f, from the pixel's depth d, camera-frame
    normal n and the mean 1/f of the live camera (Keller et al. 2013); a merge averages it with the confidence weights, as
    it does the position, and a surfel without a radius (0) takes the pixel's.  No association, merge or append
    decision depends on it: every other value of the map is what surfel_radii=False gives.  Radii carry no gradient."""
    if not isinstance(pointclouds, Pointclouds):
        raise TypeError("Expected pointclouds to be of type gradslam.Pointclouds. Got {0}.".format(type(pointclouds)))
    _check_frame(rgbdimages)
    _check_surfel_radii(surfel_radii)
    _check_fusion_inputs(pointclouds, rgbdimages)
    _check_embeddings(pointclouds, rgbdimages)
    if not inplace:
        pointclouds = pointclouds.clone()
    return _fuse(pointclouds, rgbdimages, sigma, dist_th, dot_th, radii=surfel_radii)
