"""Pointclouds: batch of variable-length surfel maps (points, normals, colors, features/confidence).

Host-side mirror of gradslam.Pointclouds (gradslam/structures/pointclouds.py:13-1467): same constructor,
list / padded views, arithmetic helpers, `append_points`, `transform`, `pinhole_projection`, `clone`,
`detach`, `to`, indexing.  The representation is different by design (SURVEY.md §8f.1): instead of the
reference's list <-> padded duality, rebuilt with `torch.cat` on every append, the map lives in ONE
capacity-backed store of SECTOR-PACKED rows that the fusion kernels update IN PLACE:

    geometry  (B, capacity, 8)  float32   (px, py, pz, nx, ny, nz, ccount, radius)   one 32-byte DRAM sector per surfel
    colours   (B, capacity, 4)  float32   (r, g, b, 0)
    counts    (2, B)            int32     ping-pong: kernels read row `cur`, write row `cur ^ 1`

so a kernel touches a surfel with two (geometry) or three (+ colour) 128-bit accesses instead of ten scalar ones
spread over four arrays.  gradslam's tensors are STRIDED VIEWS of these rows: `points_padded = geometry[:, :N, 0:3]`,
`normals_padded = geometry[:, :N, 3:6]`, `features_padded = geometry[:, :N, 6:7]` (the confidence count),
`colors_padded = colours[:, :N, 0:3]`, `radii_padded = geometry[:, :N, 7:8]` (the surfel radius: 0 unless the map
was fused with surfel_radii=True); `*_list[b]` are the same views cut at `counts[b]`.  (Features with more than
one channel are not part of the fusion path; they live in a separate dense (B, capacity, C) tensor.)  Rows >=
counts[b] are always zero inside the padded width.  A map may also carry one embedding per surfel (ConceptFusion-style
feature maps), a dense (B, capacity, D) store of float32, float16 or bfloat16 beside the rows: `embeddings_padded` /
`embeddings_list`; the fused map update merges it with the colours' weights (fusionutils.update_map_fusion).  The per-element sizes live on the device (the kernels bump them);
the host copy is refreshed lazily, only when a caller asks for a shape-dependent view.  Everything is float32: other
floating inputs are cast on construction (the kernels read raw float32 rows).
"""
from typing import List, Optional, Union

import torch

__all__ = ["Pointclouds"]

# storage types of per-surfel embeddings, and their dtype code in the C ABI (gsx_embed_merge_append)
EMBED_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}

_ATTRS = ("points", "normals", "colors", "features")
GEO_W, COL_W = 8, 4  # floats per geometry / colour row (csrc/gsx_fusion.cu)


def _f32(t, device):
    return t.to(device=device, dtype=torch.float32)


class _PruneHistory:
    """Pruning history of a batch of maps (the removal of unstable surfels, fusionutils.prune_unstable): `ring` int32
    (t_max + 2, B) on the map's device, where ring[k % (t_max + 2), b] is element b's row count after pruned step k, and
    `step`, the number of pruned steps so far (host).  Rows are appended in step order and removed by a stable
    compaction, so the rows created at step k are [ring(k - 1), ring(k)) and no per-row timestamp is stored."""

    def __init__(self, ring: torch.Tensor, step: int, t_max: int):
        self.ring, self.step, self.t_max = ring, int(step), int(t_max)

    @classmethod
    def fresh(cls, B: int, t_max: int, device):
        return cls(torch.zeros((t_max + 2, B), dtype=torch.int32, device=device), 0, t_max)

    def to(self, device):
        return _PruneHistory(self.ring.to(device, copy=True), self.step, self.t_max)


class Pointclouds(object):
    def __init__(self, points=None, normals=None, colors=None, features=None,
                 device: Union[torch.device, str, None] = None, *, embeddings=None):
        """embeddings (extension): per-surfel embeddings, of the same type as points - a list of (N_b, D) tensors or a
        (B, N, D) tensor - in float32, float16 or bfloat16 (kept in that dtype), D >= 1."""
        super().__init__()
        if not (embeddings is None or isinstance(embeddings, type(points))):
            raise TypeError("Expected embeddings to be of same type as points (%r); got %r" % (type(points),
                                                                                            type(embeddings)))
        if not (points is None or isinstance(points, list) or torch.is_tensor(points)):
            raise TypeError("Expected points to be of type list or tensor or None; got %r" % type(points))
        for name, val in (("normals", normals), ("colors", colors), ("features", features)):
            if not (val is None or isinstance(val, type(points))):
                raise TypeError("Expected %s to be of same type as points (%r); got %r" % (name, type(points), type(val)))
        if points is not None and len(points) == 0:
            raise ValueError("len(points) (= 0) should be > 0")

        self._geo = None  # (B, cap, 8) geometry rows
        self._col = None  # (B, cap, 4) colour rows, or None: no colours
        self._feat = None  # (B, cap, C) generic features (C != 1), or None
        self._has_normals = False
        self._has_cc = False  # single-channel features (the confidence count) live in slot 6 of the geometry rows
        self._counts_dev = None  # int32 (2, B): ping-pong; row self._cur is current
        self._cur = 0
        self._counts_host = None  # list[int] or None when stale
        self._bound = 0  # host-side upper bound of max(counts) (valid even when _counts_host is stale)
        self._overflow = None  # int32 device flag set by kernels if capacity was exceeded
        self._B = 0
        self._list_cache = {}
        self._uninit = False  # store was allocated without zero-fill: rows >= counts[b] may hold garbage
        self._tail_dirty = False  # the ragged tail [counts[b], max(counts)) must be zeroed before a padded view
        self._prune = None  # _PruneHistory once unstable surfels have been removed from this map (PointFusion)
        self._emb = None  # (B, cap, D) per-surfel embeddings, or None

        if isinstance(points, list):
            shapes = [p.shape for p in points]
            if any(p.ndim != 2 for p in points):
                raise ValueError("ndim of all tensors in points list should be 2")
            if any(s[-1] != 3 for s in shapes):
                raise ValueError("last dim of all tensors in points should have shape 3 (X, Y, Z)")
            self.device = torch.empty(0, device=device).device if device is not None else points[0].device
            counts = [int(s[0]) for s in shapes]
            if not (normals is None or [n.shape for n in normals] == shapes):
                raise ValueError("normals tensors should have same shape as points tensors, but didn't")
            if not (colors is None or [c.shape for c in colors] == shapes):
                raise ValueError("colors tensors should have same shape as points tensors, but didn't")
            if not (features is None or all(f.ndim == 2 for f in features)):
                raise ValueError("ndim of all tensors in features list should be 2")
            if not (features is None or [len(f) for f in features] == counts):
                raise ValueError("number of features per pointcloud has to be equal to number of points")
            if not (features is None or len(set(f.shape[-1] for f in features)) == 1):
                raise ValueError("number of features per pointcloud has to be the same")
            self._B = len(points)
            self._alloc_buffers(max(counts), normals is not None, colors is not None,
                                0 if features is None else features[0].shape[-1])
            for key, lst in zip(_ATTRS, (points, normals, colors, features)):
                if lst is None:
                    continue
                dst = self._view(key)
                for b, x in enumerate(lst):
                    if x.shape[0] > 0:
                        dst[b, : x.shape[0]] = _f32(x, self.device)
            if embeddings is not None:
                if len(embeddings) != len(points) or any(not torch.is_tensor(e) or e.ndim != 2 for e in embeddings):
                    raise ValueError("embeddings should be a list of one 2-D tensor per pointcloud")
                if [int(e.shape[0]) for e in embeddings] != counts:
                    raise ValueError("number of embeddings per pointcloud has to be equal to number of points")
                if len(set((e.shape[1], e.dtype) for e in embeddings)) != 1:
                    raise ValueError("embeddings of every pointcloud must have the same dimension and dtype")
                self._alloc_embeddings(embeddings[0].shape[1], embeddings[0].dtype, max(counts))
                for b, e in enumerate(embeddings):
                    self._emb[b, : e.shape[0]] = e.to(self.device)
            self._set_counts(counts)
        elif torch.is_tensor(points):
            self.device = torch.empty(0, device=device).device if device is not None else points.device
            if points.ndim != 3:
                raise ValueError("points should have ndim=3, but had ndim={}".format(points.ndim))
            if points.shape[-1] != 3:
                raise ValueError("last dim of points should have shape 3 (X, Y, Z) but had shape %r" % (points.shape[-1]))
            if points.shape[0] == 0:
                raise ValueError("Batch size of 0 not supported yet. Got input points shape {}.".format(points.shape))
            if not (normals is None or normals.shape == points.shape):
                raise ValueError("normals tensor should have same shape as points tensor, but didn't: %r != %r"
                                 % (normals.shape, points.shape))
            if not (colors is None or colors.shape == points.shape):
                raise ValueError("colors tensor should have same shape as points tensor, but didn't: %r != %r"
                                 % (colors.shape, points.shape))
            if not (features is None or features.ndim == 3):
                raise ValueError("features should have ndim=3, but had ndim={}".format(features.ndim))
            if not (features is None or features.shape[:-1] == points.shape[:-1]):
                raise ValueError("first 2 dims of features tensor and points tensor should have same shape, but "
                                 "didn't: %r != %r" % (features.shape[:-1], points.shape[:-1]))
            self._B = points.shape[0]
            N = points.shape[1]
            self._alloc_buffers(N, normals is not None, colors is not None,
                                0 if features is None else features.shape[-1])
            for key, t in zip(_ATTRS, (points, normals, colors, features)):
                if t is not None and N > 0:
                    self._view(key)[:, :N] = _f32(t, self.device)
            if embeddings is not None:
                if embeddings.ndim != 3 or embeddings.shape[:2] != points.shape[:2]:
                    raise ValueError("embeddings should be (B, N, D) with the points' B and N; got %r" % (
                        tuple(embeddings.shape),))
                self._alloc_embeddings(embeddings.shape[2], embeddings.dtype, N)
                self._emb[:, :N] = embeddings.to(self.device)
            self._set_counts([N] * self._B)
        else:
            if embeddings is not None:
                raise ValueError("embeddings need points")
            self.device = torch.empty(0, device=device).device if device is not None else torch.device("cpu")

    # ------------------------------------------------------------------ packed storage
    def _alloc_buffers(self, capacity: int, with_normals: bool, with_colors: bool, features_dim: int, zero: bool = True):
        alloc = torch.zeros if zero else torch.empty
        cap = max(int(capacity), 0)
        self._geo = alloc((self._B, cap, GEO_W), dtype=torch.float32, device=self.device)
        self._col = alloc((self._B, cap, COL_W), dtype=torch.float32, device=self.device) if with_colors else None
        self._has_normals = bool(with_normals)
        self._has_cc = features_dim == 1
        self._feat = (alloc((self._B, cap, int(features_dim)), dtype=torch.float32, device=self.device)
                      if features_dim > 1 else None)

    def _alloc_embeddings(self, dim, dtype, capacity=None):
        """A zeroed (B, capacity, dim) embedding store (capacity: the rows' by default)."""
        if isinstance(dim, bool) or not isinstance(dim, int) or dim < 1:
            raise ValueError("embedding dimension must be an int >= 1; got {}".format(dim))
        if dtype not in EMBED_DTYPES:
            raise TypeError("embeddings must be float32, float16 or bfloat16; got {}".format(dtype))
        cap = self.capacity if capacity is None else max(int(capacity), 0)
        self._emb = torch.zeros((self._B, cap, dim), dtype=dtype, device=self.device)

    def _buffers(self):
        return [t for t in (self._geo, self._col, self._feat, self._emb) if t is not None]

    def _view(self, key):
        """Full-capacity strided view (B, capacity, C) of one attribute, or None."""
        if self._geo is None:
            return None
        if key == "points":
            return self._geo[..., 0:3]
        if key == "normals":
            return self._geo[..., 3:6] if self._has_normals else None
        if key == "colors":
            return None if self._col is None else self._col[..., 0:3]
        if key == "features":
            return self._geo[..., 6:7] if self._has_cc else self._feat
        if key == "radii":
            return self._geo[..., 7:8]
        if key == "embeddings":
            return self._emb
        raise KeyError(key)

    def _grad_tensors(self):
        """Tensors whose requires_grad switches the fusion / ICP ops to their differentiable mode (the embeddings only
        switch the fusion's: tracking does not read them)."""
        return [t for t in (self._geo, self._col, self._feat) if t is not None]

    # ------------------------------------------------------------------ size bookkeeping
    def _set_counts(self, counts: List[int]):
        self._counts_host = [int(c) for c in counts]
        self._bound = max(self._counts_host) if self._counts_host else 0
        t = torch.tensor([self._counts_host, self._counts_host], dtype=torch.int32)
        if self.device.type == "cuda":
            # from pinned memory, asynchronously: a pageable source would synchronise the current stream, i.e. make the
            # host wait for all fusion work enqueued so far every time a map is (re)started
            t = t.pin_memory().to(self.device, non_blocking=True)
        self._counts_dev = t
        self._cur = 0
        self._list_cache = {}
        self._tail_dirty = self._uninit

    def _host_counts(self, stream=None) -> List[int]:
        """Per-element sizes on the host; synchronises with the device only if kernels changed them.  stream: read them
        (and the overflow flag) through this CUDA stream and wait for IT only - the caller has ordered it after the
        kernels that produced this map - instead of the current stream, which may already hold later work."""
        if self._counts_host is None:
            if stream is not None and self._counts_dev.is_cuda:
                with torch.cuda.stream(stream):
                    host = torch.empty(self._B + 1, dtype=torch.int32, pin_memory=True)
                    host[: self._B].copy_(self._counts_dev[self._cur], non_blocking=True)
                    if self._overflow is not None:
                        host[self._B:].copy_(self._overflow, non_blocking=True)
                    else:
                        host[self._B] = 0
                stream.synchronize()
                vals = host.tolist()
                self._counts_host = [int(c) for c in vals[: self._B]]
                self._bound = max(self._counts_host)
                if vals[self._B] != 0:
                    raise RuntimeError("gradslam_b200: surfel map capacity exceeded; points were dropped")
            else:
                self._counts_host = [int(c) for c in self._counts_dev[self._cur].tolist()]
                self._bound = max(self._counts_host)
                self._check_overflow()
        return self._counts_host

    def _check_overflow(self):
        if self._overflow is not None and int(self._overflow.item()) != 0:
            raise RuntimeError("gradslam_b200: surfel map capacity exceeded; points were dropped")

    @property
    def capacity(self) -> int:
        return 0 if self._geo is None else int(self._geo.shape[1])

    def _mark_device_updated(self, new_bound: int):
        """Called by the fusion ops after kernels wrote counts into the other ping-pong row."""
        self._cur ^= 1
        self._counts_host = None
        self._bound = min(int(new_bound), self.capacity)
        self._list_cache = {}
        self._tail_dirty = self._uninit

    def _allocate(self, B: int, capacity: int, features_dim: int = 1, zero: bool = True):
        """Turns an EMPTY object into B empty maps (points, normals, colours [, confidence]) with the given capacity
        (used by the fusion ops).  zero=False skips the fill: the kernels never read rows >= counts[b]; the zero
        padding that the `*_padded` views promise is then restored lazily, only for the ragged tail (see _padded)."""
        assert not self.has_points
        self._B = int(B)
        self._alloc_buffers(capacity, True, True, features_dim, zero)
        self._uninit = not zero
        self._set_counts([0] * self._B)

    def _attach(self, geo: torch.Tensor, col: torch.Tensor, uninit: bool = True):
        """Turns an EMPTY object into B empty maps that live in caller-provided row arrays - geometry rows (B, cap, 8)
        and colour rows (B, cap, 4), dense float32 - e.g. one rank's block of a job-wide store (parallel.GatheredMaps)."""
        assert not self.has_points
        if geo.shape[:2] != col.shape[:2] or geo.shape[2] != GEO_W or col.shape[2] != COL_W:
            raise ValueError("row arrays must be (B, cap, %d) and (B, cap, %d); got %r and %r" % (
                GEO_W, COL_W, tuple(geo.shape), tuple(col.shape)))
        if not (geo.is_contiguous() and col.is_contiguous() and geo.dtype == col.dtype == torch.float32):
            raise ValueError("row arrays must be dense float32")
        self.device = geo.device
        self._B = int(geo.shape[0])
        self._geo, self._col, self._feat = geo, col, None
        self._has_normals = self._has_cc = True
        self._uninit = bool(uninit)
        self._set_counts([0] * self._B)

    def _overflow_flag(self):
        if self._overflow is None:
            self._overflow = torch.zeros(1, dtype=torch.int32, device=self.device)
        return self._overflow

    def reserve(self, capacity: int):
        """Grows every buffer to at least `capacity` rows (amortised doubling, zero-filled)."""
        cap = self.capacity
        if capacity <= cap:
            return
        new_cap = max(int(capacity), 2 * cap)

        def grow(st):
            if st is None:
                return None
            grown = torch.zeros((st.shape[0], new_cap, st.shape[2]), dtype=st.dtype, device=st.device)
            if cap > 0:
                grown[:, :cap] = st  # (a dirty tail, if any, is copied too and stays flagged)
            return grown

        self._geo, self._col, self._feat = grow(self._geo), grow(self._col), grow(self._feat)
        self._emb = grow(self._emb)
        self._list_cache = {}

    # ------------------------------------------------------------------ protocol
    def __len__(self):
        return self._B

    @property
    def has_points(self):
        return self._geo is not None

    @property
    def has_normals(self):
        return self._geo is not None and self._has_normals

    @property
    def has_colors(self):
        return self._col is not None

    @property
    def has_features(self):
        return self._geo is not None and (self._has_cc or self._feat is not None)

    @property
    def has_embeddings(self):
        return self._geo is not None and self._emb is not None

    @property
    def embedding_dim(self):
        """D of the per-surfel embeddings, 0 without."""
        return int(self._emb.shape[2]) if self.has_embeddings else 0

    @property
    def num_features(self):
        if not self.has_features:
            return 0
        return 1 if self._has_cc else self._feat.shape[-1]

    @property
    def num_points_per_pointcloud(self):
        if not self.has_points:
            return torch.tensor([0], device=self.device)
        return self._counts_dev[self._cur].to(torch.int64)

    @property
    def equisized(self):
        if not self.has_points:
            return None
        return len(set(self._host_counts())) == 1

    @property
    def _N(self):
        return max(self._host_counts()) if self.has_points else 0

    def _zero_tail(self, n: int):
        counts = self._host_counts()
        for st in self._buffers():
            for b, c in enumerate(counts):
                if c < n:
                    st[b, c:n].zero_()

    def _clean_tail(self):
        """Zeroes rows [counts[b], max(counts)) of every buffer (only needed after a zero=False allocation)."""
        if self._tail_dirty and self.has_points:
            self._zero_tail(self._N)
            self._tail_dirty = False

    def _zero_rows_upto(self, n: int):
        """Zeroes rows [counts[b], n) of every buffer (padding contract for an externally chosen width)."""
        if self._uninit:  # zero-initialised stores already satisfy the contract
            self._zero_tail(n)

    def _padded(self, key):
        st = self._view(key)
        if st is None:
            return None
        self._clean_tail()
        return st[:, : self._N]

    def _list(self, key):
        st = self._view(key)
        if st is None:
            return None
        if key not in self._list_cache:
            self._list_cache[key] = [st[b, :c] for b, c in enumerate(self._host_counts())]
        return self._list_cache[key]

    points_padded = property(lambda self: self._padded("points"))
    normals_padded = property(lambda self: self._padded("normals"))
    colors_padded = property(lambda self: self._padded("colors"))
    features_padded = property(lambda self: self._padded("features"))
    points_list = property(lambda self: self._list("points"))
    normals_list = property(lambda self: self._list("normals"))
    colors_list = property(lambda self: self._list("colors"))
    features_list = property(lambda self: self._list("features"))
    # surfel radii (B, N, 1) / [(N_b, 1)]: written by the fused map update with surfel_radii=True, 0 otherwise; they carry
    # no gradient through the fusion ops
    radii_padded = property(lambda self: self._padded("radii"))
    radii_list = property(lambda self: self._list("radii"))
    # per-surfel embeddings (B, N, D) / [(N_b, D)] in their storage dtype, or None
    embeddings_padded = property(lambda self: self._padded("embeddings"))
    embeddings_list = property(lambda self: self._list("embeddings"))

    @property
    def nonpad_mask(self):
        if not self.has_points:
            return None
        c = self._counts_dev[self._cur].to(torch.int64).view(-1, 1)
        return torch.arange(self._N, device=self.device).view(1, -1) < c

    # ------------------------------------------------------------------ setters (shape-preserving, as pointclouds.py:811-946)
    def _assert_set_padded(self, value, first_2_dims_only=False):
        if not torch.is_tensor(value):
            raise TypeError("value must be torch.Tensor. Got {}".format(type(value)))
        if not self.has_points:
            raise ValueError("cannot set padded representation for an empty pointclouds object")
        if self.device != torch.empty(0, device=value.device).device:
            raise ValueError("value must have the same device as pointclouds object: {} vs {}".format(
                value.device, self.device))
        if value.ndim != 3:
            raise ValueError("value.ndim should be 3. Got {}".format(value.ndim))
        exp = (self._B, self._N) if first_2_dims_only else (self._B, self._N, 3)
        got = tuple(value.shape[:2]) if first_2_dims_only else tuple(value.shape)
        if got != exp:
            raise ValueError("Expected value to have shape {}. Got {}".format(exp, tuple(value.shape)))

    def _writable_view(self, key, channels: int):
        """Fresh (out-of-place, autograd friendly: never mutate a tensor a caller may still hold) full-capacity view of
        attribute `key` with `channels` channels, creating / re-shaping its buffer if needed."""
        cap = max(self.capacity, self._N)
        if key in ("points", "normals", "radii") or (key == "features" and channels == 1):
            self._geo = self._geo.clone()
            if key == "normals":
                self._has_normals = True
            if key == "features":
                self._has_cc, self._feat = True, None
        elif key == "colors":
            self._col = (torch.zeros((self._B, cap, COL_W), dtype=torch.float32, device=self.device)
                         if self._col is None else self._col.clone())
        else:  # features with C != 1
            if self._has_cc:
                self._geo = self._geo.clone()
                self._geo[..., 6] = 0
                self._has_cc = False
            self._feat = torch.zeros((self._B, cap, channels), dtype=torch.float32, device=self.device)
        self._list_cache = {}
        return self._view(key)

    def _set_padded(self, key, value, first_2=False):
        self._assert_set_padded(value, first_2)
        n = self._N
        dst = self._writable_view(key, value.shape[-1])
        dst[:, :n] = _f32(value, self.device)

    def _assert_set_list(self, value, first_dim_only=False):
        if not isinstance(value, list):
            raise TypeError("value must be list of tensors. Got {}".format(type(value)))
        if not self.has_points:
            raise ValueError("cannot set list representation for an empty pointclouds object")
        if len(value) != self._B:
            raise ValueError("Expected value to have len {}. Got {}".format(self._B, len(value)))
        for b, (v, c) in enumerate(zip(value, self._host_counts())):
            if not torch.is_tensor(v):
                raise TypeError("value must be list of tensors")
            if v.ndim != 2 or v.shape[0] != c or (not first_dim_only and v.shape[1] != 3):
                raise ValueError("Shape of tensor {} in value does not match pointcloud {}".format(b, b))

    def _set_list(self, key, value, first_dim_only=False):
        self._assert_set_list(value, first_dim_only)
        dst = self._writable_view(key, value[0].shape[-1])
        for b, v in enumerate(value):
            dst[b, : v.shape[0]] = _f32(v, self.device)

    points_padded = points_padded.setter(lambda self, v: self._set_padded("points", v))
    normals_padded = normals_padded.setter(lambda self, v: self._set_padded("normals", v))
    colors_padded = colors_padded.setter(lambda self, v: self._set_padded("colors", v))
    features_padded = features_padded.setter(lambda self, v: self._set_padded("features", v, True))
    points_list = points_list.setter(lambda self, v: self._set_list("points", v))
    normals_list = normals_list.setter(lambda self, v: self._set_list("normals", v))
    colors_list = colors_list.setter(lambda self, v: self._set_list("colors", v))
    features_list = features_list.setter(lambda self, v: self._set_list("features", v, True))
    radii_padded = radii_padded.setter(lambda self, v: self._set_radii_padded(v))
    radii_list = radii_list.setter(lambda self, v: self._set_radii_list(v))
    embeddings_padded = embeddings_padded.setter(lambda self, v: self._set_embeddings_padded(v))
    embeddings_list = embeddings_list.setter(lambda self, v: self._set_embeddings_list(v))

    def _fresh_embeddings(self, dim, dtype):
        """A new (never a tensor a caller may hold) zeroed store for the setters."""
        cap = max(self.capacity, self._N)
        self._alloc_embeddings(dim, dtype, cap)
        self._list_cache = {}
        return self._emb

    def _set_embeddings_padded(self, value):
        self._assert_set_padded(value, True)
        dst = self._fresh_embeddings(value.shape[-1], value.dtype)
        dst[:, : self._N] = value

    def _set_embeddings_list(self, value):
        self._assert_set_list(value, True)
        if len(set((v.shape[1], v.dtype) for v in value)) != 1:
            raise ValueError("embeddings of every pointcloud must have the same dimension and dtype")
        dst = self._fresh_embeddings(value[0].shape[1], value[0].dtype)
        for b, v in enumerate(value):
            dst[b, : v.shape[0]] = v

    def _set_radii_padded(self, value):
        self._assert_set_padded(value, True)
        if value.shape[-1] != 1:
            raise ValueError("radii must have one channel. Got {}".format(value.shape[-1]))
        self._set_padded("radii", value, True)

    def _set_radii_list(self, value):
        self._assert_set_list(value, True)
        if any(v.shape[1] != 1 for v in value):
            raise ValueError("radii must have one channel")
        self._set_list("radii", value, True)

    # ------------------------------------------------------------------ indexing
    def __getitem__(self, index):
        if not self.has_points:
            raise IndexError("Cannot index empty pointclouds object")
        if isinstance(index, int):
            idx = [index]
        elif isinstance(index, slice):
            idx = list(range(self._B))[index]
        elif isinstance(index, list):
            idx = index
        elif isinstance(index, torch.Tensor):
            if index.dim() != 1 or index.dtype.is_floating_point:
                raise IndexError(index)
            idx = index.nonzero().flatten().tolist() if index.dtype == torch.bool else index.tolist()
        else:
            raise IndexError(index)
        pick = lambda lst: None if lst is None else [lst[i] for i in idx]
        return Pointclouds(points=pick(self.points_list), normals=pick(self.normals_list),
                           colors=pick(self.colors_list), features=pick(self.features_list),
                           embeddings=pick(self.embeddings_list))

    # ------------------------------------------------------------------ arithmetic helpers (pointclouds.py:303-614)
    def __add__(self, other):
        try:
            return self.clone().offset_(other)
        except TypeError:
            raise NotImplementedError("Pointclouds + {} currently not implemented.".format(type(other)))

    def __sub__(self, other):
        try:
            return self.clone().offset_(other * -1)
        except TypeError:
            raise NotImplementedError("Pointclouds - {} currently not implemented.".format(type(other)))

    def __mul__(self, other):
        try:
            return self.clone().scale_(other)
        except TypeError:
            raise NotImplementedError("Pointclouds * {} currently not implemented.".format(type(other)))

    def __truediv__(self, other):
        try:
            return self.__mul__(1.0 / other)
        except TypeError:
            raise NotImplementedError("Pointclouds / {} currently not implemented.".format(type(other)))

    def __matmul__(self, other):
        if not torch.is_tensor(other):
            raise NotImplementedError("Pointclouds @ {} currently not implemented.".format(type(other)))
        if not ((other.ndim == 2 or other.ndim == 3) and (other.shape[-2:] == (3, 3) or other.shape[-2:] == (4, 4))):
            raise ValueError(
                "Unsupported shape for Pointclouds @ operand: {}\nUse tensor of shape (3, 3) or (B, 3, 3) for "
                "rotations, or (4, 4) or (B, 4, 4) for transformations".format(other.shape))
        if other.shape[-2:] == (3, 3):
            return self.clone().rotate_(other, pre_multiplication=False)
        return self.clone().transform_(other, pre_multiplication=False)

    def rotate(self, rmat, *, pre_multiplication=True):
        return self.clone().rotate_(rmat, pre_multiplication=pre_multiplication)

    def transform(self, transform, *, pre_multiplication=True):
        return self.clone().transform_(transform, pre_multiplication=pre_multiplication)

    def pinhole_projection(self, intrinsics):
        return self.clone().pinhole_projection_(intrinsics)

    def _write_padded(self, key, value):
        n = self._N
        self._writable_view(key, value.shape[-1])[:, :n] = value

    def offset_(self, offset):
        if not (torch.is_tensor(offset) or isinstance(offset, (float, int))):
            raise TypeError("Operand should be tensor, float or int but was %r instead" % type(offset))
        if not self.has_points:
            return self
        mask = self.nonpad_mask.to(self.points_padded.dtype).unsqueeze(-1)
        self._write_padded("points", self.points_padded + offset * mask)
        return self

    def scale_(self, scale):
        if not (torch.is_tensor(scale) or isinstance(scale, (float, int))):
            raise TypeError("Operand should be tensor, float or int but was %r instead" % type(scale))
        if not self.has_points:
            return self
        mask = self.nonpad_mask.to(self.points_padded.dtype).unsqueeze(-1)
        self._write_padded("points", self.points_padded * scale * mask)
        return self

    def rotate_(self, rmat, *, pre_multiplication=True):
        if not torch.is_tensor(rmat):
            raise TypeError("Rotation matrix should be tensor, but was %r instead" % type(rmat))
        if not ((rmat.ndim == 2 or rmat.ndim == 3) and rmat.shape[-2:] == (3, 3)):
            raise ValueError("Rotation matrix should be of shape (3, 3) or (B, 3, 3), but was {} instead.".format(
                rmat.shape))
        if rmat.ndim == 3 and rmat.shape[0] != self._B:
            raise ValueError("Rotation matrix batch size ({}) != Pointclouds batch size ({})".format(
                rmat.shape[0], self._B))
        if not self.has_points:
            return self
        if pre_multiplication:
            rmat = rmat.transpose(-1, -2)
        eq = "bij,jk->bik" if rmat.ndim == 2 else "bij,bjk->bik"
        self._write_padded("points", torch.einsum(eq, self.points_padded, rmat))
        if self.has_normals:
            self._write_padded("normals", torch.einsum(eq, self.normals_padded, rmat))
        return self

    def transform_(self, transform, *, pre_multiplication=True):
        if not torch.is_tensor(transform):
            raise TypeError("transform should be tensor, but was %r instead" % type(transform))
        if not ((transform.ndim == 2 or transform.ndim == 3) and transform.shape[-2:] == (4, 4)):
            raise ValueError("transform should be of shape (4, 4) or (B, 4, 4), but was {} instead.".format(
                transform.shape))
        if transform.ndim == 3 and transform.shape[0] != self._B:
            raise ValueError("transform batch size ({}) != Pointclouds batch size ({})".format(
                transform.shape[0], self._B))
        if not self.has_points:
            return self
        rmat = transform[..., :3, :3]
        tvec = transform[..., :3, 3]
        while tvec.ndim < 3:
            tvec = tvec.unsqueeze(-2)
        return self.rotate_(rmat, pre_multiplication=pre_multiplication).offset_(tvec)

    def pinhole_projection_(self, intrinsics):
        if not torch.is_tensor(intrinsics):
            raise TypeError("intrinsics should be tensor, but was {} instead".format(type(intrinsics)))
        if not ((intrinsics.ndim == 2 or intrinsics.ndim == 3) and intrinsics.shape[-2:] == (4, 4)):
            raise ValueError("intrinsics should be of shape (4, 4) or (B, 4, 4), but was {} instead.".format(
                intrinsics.shape))
        if not self.has_points:
            return self
        from ..geometry import projutils

        uv = projutils.project_points(self.points_padded, intrinsics)
        mask = self.nonpad_mask.to(uv.dtype).unsqueeze(-1)
        self._write_padded("points", projutils.homogenize_points(uv) * mask)
        return self

    # ------------------------------------------------------------------ copies / device moves
    def _like(self, fn):
        other = Pointclouds(device=self.device)
        if not self.has_points:
            return other
        other._B = self._B
        keep = max(self._N, 1)  # copy the populated rows only (one sync beats cloning gigabytes of spare capacity)
        cp = lambda st: None if st is None else fn(st[:, :keep])
        other._geo, other._col, other._feat = cp(self._geo), cp(self._col), cp(self._feat)
        other._emb = cp(self._emb)
        other._has_normals, other._has_cc = self._has_normals, self._has_cc
        other.device = other._geo.device
        other._counts_dev = self._counts_dev.clone().to(other.device)
        other._cur = self._cur
        other._counts_host = None if self._counts_host is None else list(self._counts_host)
        other._bound = min(self._bound, keep)
        other._overflow = None if self._overflow is None else self._overflow.clone().to(other.device)
        other._uninit, other._tail_dirty = self._uninit, self._tail_dirty
        other._prune = None if self._prune is None else self._prune.to(other.device)
        return other

    def clone(self):
        return self._like(lambda t: t.clone())

    def detach(self):
        return self._like(lambda t: t.detach().clone())

    def to(self, device, copy: bool = False):
        device = torch.empty(0, device=device).device
        if not copy and self.device == device:
            return self
        other = self._like(lambda t: t.to(device, copy=True))
        other.device = device
        return other

    def download(self, out: Optional["Pointclouds"] = None, stream=None) -> "Pointclouds":
        """Asynchronous read-back of the populated rows into PINNED host memory: returns a CPU Pointclouds (same packed
        layout) whose buffers are filled by device-to-host copies enqueued on `stream` (default: the current stream) -
        synchronise that stream before touching the result.  Pass the previous result as `out` to re-use its pinned
        buffers.  One host synchronisation (the map sizes, read through `stream`) precedes the copies."""
        if not self.has_points:
            return Pointclouds()
        counts = self._host_counts(stream)
        n = max(max(counts), 1)
        if out is None or out._geo is None or out._geo.shape[1] < n or out._B != self._B:
            cap = int(n * 1.05) + 1
            out = Pointclouds()
            out._B = self._B
            pin = lambda st: None if st is None else torch.zeros((st.shape[0], cap, st.shape[2]), dtype=st.dtype,
                                                                 pin_memory=True)
            out._geo, out._col, out._feat = pin(self._geo), pin(self._col), pin(self._feat)
        if self._emb is not None and (out._emb is None or out._emb.shape[1] < n or out._emb.shape[2] != self._emb.shape[2]
                                      or out._emb.dtype != self._emb.dtype):
            out._emb = torch.zeros((self._B, out._geo.shape[1], self._emb.shape[2]), dtype=self._emb.dtype,
                                   pin_memory=True)
        elif self._emb is None:
            out._emb = None
        out._has_normals, out._has_cc = self._has_normals, self._has_cc
        ctx = torch.cuda.stream(stream) if stream is not None else torch.cuda.device(self.device)
        with ctx:
            for dst, src in ((out._geo, self._geo), (out._col, self._col), (out._feat, self._feat),
                             (out._emb, self._emb)):
                if src is None:
                    continue
                for b, c in enumerate(counts):
                    if c > 0:
                        dst[b, :c].copy_(src[b, :c], non_blocking=True)
        out._set_counts(counts)
        out._uninit, out._tail_dirty = True, True  # (rows of a previous, longer download may remain beyond counts[b])
        return out

    def cpu(self):
        return self.to(torch.device("cpu"))

    def cuda(self):
        return self.to(torch.device("cuda"))

    # ------------------------------------------------------------------ export for visualisation (host side)
    def open3d(self, index: int, include_colors: bool = True, max_num_points: Optional[int] = None,
               include_normals: bool = False):
        """`open3d.geometry.PointCloud` of cloud `index` (pointclouds.py:1239-1297); needs the open3d package."""
        from .export import to_open3d

        return to_open3d(self, index, include_colors, max_num_points, include_normals)

    def plotly(self, index: int, include_colors: bool = True, max_num_points: Optional[int] = 200000,
               as_figure: bool = True, point_size: int = 2):
        """plotly Figure / Scatter3d of cloud `index` (pointclouds.py:1299-1383); needs the plotly package."""
        from .export import to_plotly

        return to_plotly(self, index, include_colors, max_num_points, as_figure, point_size)

    # ------------------------------------------------------------------ growth
    def _adopt(self, src: "Pointclouds"):
        self._geo, self._col, self._feat, self._B = src._geo, src._col, src._feat, src._B
        self._emb = src._emb
        self._has_normals, self._has_cc = src._has_normals, src._has_cc
        self._counts_dev, self._cur = src._counts_dev, src._cur
        self._counts_host, self._bound, self._overflow = src._counts_host, src._bound, src._overflow
        self._uninit, self._tail_dirty = src._uninit, src._tail_dirty
        self._prune = src._prune
        self._list_cache = {}

    def append_points(self, pointclouds: "Pointclouds"):
        """Appends another batch of clouds element-wise, in place (pointclouds.py:1117-1237)."""
        if not isinstance(pointclouds, type(self)):
            raise TypeError("Append object must be of type gradslam.Pointclouds, but was of type {}.".format(
                type(pointclouds)))
        if not (pointclouds.device == self.device):
            raise ValueError("Device of pointclouds to append and to be appended must match: ({0} != {1})".format(
                pointclouds.device, self.device))
        if not pointclouds.has_points:
            return self
        if not self.has_points:
            self._adopt(pointclouds.clone())
            return self
        if len(pointclouds) != len(self):
            raise ValueError("Batch size of pointclouds to append and to be appended must match: ({0} != {1})".format(
                len(pointclouds), len(self)))
        for what in ("normals", "colors", "features"):
            mine, theirs = getattr(self, "has_" + what), getattr(pointclouds, "has_" + what)
            if mine != theirs:
                raise ValueError("pointclouds to append and to be appended must either both have or not have {}: "
                                 "({} != {})".format(what, theirs, mine))
        if self.has_features and self.num_features != pointclouds.num_features:
            raise ValueError("pointclouds to append and to be appended must have the same number of features: "
                             "({0} != {1})".format(pointclouds.num_features, self.num_features))
        if self.has_embeddings != pointclouds.has_embeddings:
            raise ValueError("pointclouds to append and to be appended must either both have or not have embeddings: "
                             "({} != {})".format(pointclouds.has_embeddings, self.has_embeddings))
        if self.has_embeddings and (self._emb.shape[2], self._emb.dtype) != (pointclouds._emb.shape[2],
                                                                            pointclouds._emb.dtype):
            raise ValueError("pointclouds to append and to be appended must have embeddings of the same dimension and "
                             "dtype")
        mine, theirs = self._host_counts(), pointclouds._host_counts()
        total = [a + b for a, b in zip(mine, theirs)]
        self.reserve(max(total))
        for dst, src in ((self._geo, pointclouds._geo), (self._col, pointclouds._col),
                         (self._feat, pointclouds._feat), (self._emb, pointclouds._emb)):
            if dst is None:
                continue
            for b in range(self._B):
                if theirs[b] > 0:
                    dst[b, mine[b]: total[b]] = src[b, : theirs[b]]
        self._set_counts(total)
        return self
