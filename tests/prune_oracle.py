"""CPU oracle of the removal of unstable surfels (Keller et al. 2013, section 4.3), built on gsx_oracle's fusion step.

It tracks an explicit creation step per row instead of the ring of row counts the CUDA path keeps, so that the ring
arithmetic is checked against an independent formulation:

    creation step   the first pruned step after which the row is in the map (rows present when pruning starts, and rows
                    added between steps by append_points, are stamped at the next pruned step)
    pruned step s   after the fusion of step s: when s >= t_max, remove the rows created at step s - t_max whose
                    confidence is below c_stable; every other row keeps its order (an index_select, so the oracle's
                    autograd gives the gradient of the removal)

`RingPruner` restates the ring formulation of the kernel in plain Python; the CPU tests check that the two agree."""
import math

import torch

import gsx_oracle as oracle

F32 = torch.float32


class PrunedMap:
    """A gsx_oracle.SurfelMap plus the creation step of every row (per element, int64) and the pruned-step counter."""

    def __init__(self, smap=None):
        self.smap = oracle.SurfelMap() if smap is None else smap
        self.created = None
        self.step = 0

    def counts(self):
        return self.smap.counts() if self.smap.has_points else []


def prune_step(pm, c_stable, t_max):
    """One pruned step, in place.  Returns the kept row indices per element (None for a map without rows)."""
    s = pm.step
    pm.step += 1
    m = pm.smap
    if not m.has_points:
        return None
    if pm.created is None:
        pm.created = [torch.empty(0, dtype=torch.int64) for _ in range(m.B)]
    keeps = []
    for b in range(m.B):
        n_new = m.points[b].shape[0] - pm.created[b].shape[0]
        pm.created[b] = torch.cat([pm.created[b], torch.full((n_new,), s, dtype=torch.int64)])
        remove = torch.zeros(m.points[b].shape[0], dtype=torch.bool)
        if s >= t_max:
            remove = (pm.created[b] == s - t_max) & (m.ccounts[b][:, 0] < torch.tensor(c_stable, dtype=F32))
        keep = torch.nonzero(~remove).flatten()
        keeps.append(keep)
        m.points[b], m.normals[b] = m.points[b][keep], m.normals[b][keep]
        m.colors[b], m.ccounts[b] = m.colors[b][keep], m.ccounts[b][keep]
        pm.created[b] = pm.created[b][keep]
    return keeps


class RingPruner:
    """The kernel's formulation: ring[k % (t_max + 2)][b] = row count after pruned step k, ring(-1) = 0; the window of
    step s is [ring(s - t_max - 1), ring(s - t_max)) (for t_max = 0 the window ends at the current count)."""

    def __init__(self, B, t_max):
        self.t_max, self.R = t_max, t_max + 2
        self.ring = [[0] * B for _ in range(self.R)]
        self.step = 0

    def at(self, k, b):
        return 0 if k < 0 else self.ring[k % self.R][b]

    def __call__(self, smap, c_stable):
        s, t = self.step, self.t_max
        self.step += 1
        if not smap.has_points:
            return
        for b in range(smap.B):
            count = smap.points[b].shape[0]
            ws = min(self.at(s - t - 1, b), count) if s >= t else count
            we = (count if t == 0 else min(self.at(s - t, b), count)) if s >= t else count
            idx = torch.arange(count)
            remove = (idx >= ws) & (idx < we) & (smap.ccounts[b][:, 0] < torch.tensor(c_stable, dtype=F32))
            keep = torch.nonzero(~remove).flatten()
            smap.points[b], smap.normals[b] = smap.points[b][keep], smap.normals[b][keep]
            smap.colors[b], smap.ccounts[b] = smap.colors[b][keep], smap.ccounts[b][keep]
            removed = int(remove.sum())
            for k in range(max(s - t, 0), s):
                self.ring[k % self.R][b] -= removed
            self.ring[s % self.R][b] = count - removed


def run_pointfusion(rgb, depth, K, poses=None, *, c_stable=None, t_max=None, odom="gt", dist_th=0.05, angle_th=20.0,
                    sigma=0.6, dsratio=4, numiters=20, damp=1e-8, dist_thresh=None, lambda_max=2.0, B=1.0, B2=1.0,
                    nu=200.0, association="nn", pm=None, s_begin=0):
    """gsx_oracle.run_slam(mode='pointfusion') with a pruned step after every fusion (c_stable None: no pruning).
    association: the ICP odometry's ('nn' or 'projective', tests/projective_oracle.py).  pm continues an existing
    PrunedMap from frame s_begin (the step API after a shorter call).  Returns
    (PrunedMap, poses (B,L,4,4))."""
    Bn, L, H, W, _ = depth.shape
    dot_th = math.cos(angle_th * math.pi / 180)
    kw = dict(numiters=numiters, damp=damp, dist_thresh=dist_thresh)
    if odom == "gradicp":
        kw.update(lambda_max=lambda_max, B=B, B2=B2, nu=nu)
    pm = PrunedMap() if pm is None else pm
    out_poses = torch.empty(Bn, L, 4, 4)
    K4 = K[:, 0]
    prev_pose = None
    for s in range(s_begin, L):
        d, c = depth[:, s:s + 1], rgb[:, s:s + 1]
        if s == 0 or odom == "gt":
            pose = torch.eye(4).repeat(Bn, 1, 1) if (poses is None and s == 0) else poses[:, s]
        else:
            at_prev = oracle.frame_maps(d, K, prev_pose.unsqueeze(1))
            if association == "projective":
                import projective_oracle

                pose = projective_oracle.odometry_projective(pm.smap, at_prev, prev_pose, K4, H, W, odom, dsratio, kw)
            else:
                pose = oracle.odometry(pm.smap, at_prev, prev_pose, K4, H, W, odom, dsratio, kw)
        maps = oracle.frame_maps(d, K, pose.unsqueeze(1))
        pm.smap = oracle.update_map_fusion(pm.smap, maps, c, pose, K4, dist_th, dot_th, sigma)
        if c_stable is not None:
            prune_step(pm, c_stable, t_max)
        prev_pose = pose
        out_poses[:, s] = pose
    return pm, out_poses


def confidence_quantile(smap, q):
    """Quantile q of the confidences of every row of a SurfelMap (how a threshold is chosen for a scene): the value of
    a row, so that rows whose confidence equals the threshold exist."""
    return float(torch.quantile(torch.cat([c[:, 0] for c in smap.ccounts]).detach().double(), q,
                                interpolation="lower"))
