"""CPU oracle of the removal of free-space violations (Keller et al. 2013, section 4.3, second rule), built on gsx_oracle's
fusion step and on prune_oracle's creation-step stamps.

    bound image     after the fusion of step s: pixel u of element b has a bound iff the unique correspondence table of
                    the step (gsx_oracle.find_correspondences, the "merged into" record) pairs u with row m and row m's
                    ccount after the merge is >= c_stable; the bound is z of T_s^-1 p_m (project_map's arithmetic)
    violator        a row that find_active_map_points puts at a pixel u with a bound and project_map's z <
                    bound(u) - margin (the difference rounded to fp32)
    pruned step s   removes the union of the violators and the rows prune_oracle's age rule removes, in order (an
                    index_select, so the oracle's autograd gives the gradient of the removal)

`PositionalRingPruner` restates the kernel's ring update: after a step that removes rows anywhere, ring(k) for k in
[s - t_max, s - 1] is the number of kept rows whose old index was below the old ring(k), and ring(s) the new count.  The
CPU tests check it against the creation-step formulation."""
import math

import torch

import gsx_oracle as oracle
import prune_oracle as po

F32 = torch.float32


def bound_image(smap, pc2im, pose, K, H, W, c_stable):
    """float32 (B,H,W): the bound of every pixel, -inf where there is none.  smap is the map after the merge that pc2im
    describes; pose (B,4,4) camera-to-world, K (B,4,4)."""
    bound = torch.full((smap.B, H, W), -math.inf, dtype=F32)
    if not smap.has_points or pc2im.shape[0] == 0:
        return bound
    with torch.no_grad():
        pts, _, _, cc = smap.padded()
        _, _, z = oracle.project_map(pts, pose, K)
        b, n, h, w = pc2im.unbind(1)
        stable = cc[b, n, 0] >= torch.tensor(c_stable, dtype=F32)
        bound[b[stable], h[stable], w[stable]] = z[b, n][stable]
    return bound


def violators(smap, bound, pose, K, margin):
    """Per element, bool (N_b,): the rows in front of their pixel's bound by more than margin."""
    B, H, W = bound.shape
    out = [torch.zeros(c, dtype=torch.bool) for c in smap.counts()]
    with torch.no_grad():
        table = oracle.find_active_map_points(smap, pose, K, H, W)
        if table.shape[0] == 0:
            return out
        _, _, z = oracle.project_map(smap.padded()[0], pose, K)
        b, n, h, w = table.unbind(1)
        hit = z[b, n] < bound[b, h, w] - torch.tensor(margin, dtype=F32)
        for i in range(B):
            out[i][n[(b == i) & hit]] = True
    return out


def prune_step(pm, c_stable, t_max, extra=None):
    """prune_oracle.prune_step that also removes the rows flagged in extra[b] (None: the age rule alone).  In place;
    returns the kept row indices per element (None for a map without rows)."""
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
        if extra is not None:
            remove = remove | extra[b]
        keep = torch.nonzero(~remove).flatten()
        keeps.append(keep)
        m.points[b], m.normals[b] = m.points[b][keep], m.normals[b][keep]
        m.colors[b], m.ccounts[b] = m.colors[b][keep], m.ccounts[b][keep]
        pm.created[b] = pm.created[b][keep]
    return keeps


class PositionalRingPruner(po.RingPruner):
    """The kernel's ring formulation with removals anywhere in the map (prune_oracle.RingPruner's window, plus the rows
    flagged in `extra`): every ring entry of steps s - t_max .. s - 1 moves to the position of the row it points at."""

    def __call__(self, smap, c_stable, extra=None):
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
            if extra is not None:
                remove = remove | extra[b]
            keep = torch.nonzero(~remove).flatten()
            smap.points[b], smap.normals[b] = smap.points[b][keep], smap.normals[b][keep]
            smap.colors[b], smap.ccounts[b] = smap.colors[b][keep], smap.ccounts[b][keep]
            for k in range(max(s - t, 0), s):
                old = self.ring[k % self.R][b]
                self.ring[k % self.R][b] = int((~remove[:old]).sum())
            self.ring[s % self.R][b] = int(keep.numel())


def run_pointfusion(rgb, depth, K, poses=None, *, c_stable=None, t_max=None, margin=None, odom="gt", dist_th=0.05,
                    angle_th=20.0, sigma=0.6, dsratio=4, numiters=20, damp=1e-8, dist_thresh=None, lambda_max=2.0,
                    B=1.0, B2=1.0, nu=200.0, association="nn", pm=None, s_begin=0):
    """prune_oracle.run_pointfusion with the free-space rule in every pruned step (margin None: the age rule alone,
    which is prune_oracle's run bit for bit).  Returns (PrunedMap, poses (B,L,4,4))."""
    Bn, L, H, W, _ = depth.shape
    dot_th = math.cos(angle_th * math.pi / 180)
    kw = dict(numiters=numiters, damp=damp, dist_thresh=dist_thresh)
    if odom == "gradicp":
        kw.update(lambda_max=lambda_max, B=B, B2=B2, nu=nu)
    pm = po.PrunedMap() if pm is None else pm
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
        table = oracle.find_correspondences(pm.smap, maps, pose, K4, dist_th, dot_th)
        pm.smap = oracle.fuse_with_map(pm.smap, maps, c, table, sigma)
        if c_stable is not None:
            extra = None
            if margin is not None:
                bound = bound_image(pm.smap, table, pose.detach(), K4, H, W, c_stable)
                extra = violators(pm.smap, bound, pose.detach(), K4, margin)
            prune_step(pm, c_stable, t_max, extra)
        prev_pose = pose
        out_poses[:, s] = pose
    return pm, out_poses


def rows_in_box(smap, center, half_extents, pad=0.0, motion_scale=1.0, yaw0=0.0):
    """Per element, the number of rows whose point lies inside the axis-aligned room-frame box (grown by `pad`) of
    synthetic.make_dynamic_sequence; the map's world frame is camera 0 of the element."""
    from gradslam_b200.synthetic import _room_from_cam

    out = []
    for b in range(smap.B):
        T0 = torch.from_numpy(_room_from_cam(0, b, motion_scale, yaw0)).to(torch.float64)
        p = smap.points[b].detach().double()
        room = p @ T0[:3, :3].T + T0[:3, 3]
        lo = torch.tensor(center, dtype=torch.float64) - torch.tensor(half_extents, dtype=torch.float64) - pad
        hi = torch.tensor(center, dtype=torch.float64) + torch.tensor(half_extents, dtype=torch.float64) + pad
        out.append(int(((room >= lo) & (room <= hi)).all(-1).sum()))
    return out
