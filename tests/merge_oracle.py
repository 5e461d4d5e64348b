"""CPU oracle of the merging of overlapping surfels (Keller et al. 2013, section 4.3, third rule), built on
free_space_oracle and radii_oracle, which it leaves as they are.  The radius column rides beside the SurfelMap, per
element a float32 (N_b, 1) tensor, as in radii_oracle.

    absorber        after the fusion of step s, pixel u of element b whose correspondence-table row pairs it with row m,
                    where m's ccount after the merge is >= c_stable (the pixels that have a free-space bound), unless
                    the free-space rule removes m in this step
    candidate       a row n that find_active_map_points puts at u with n != m, no table row pairing any pixel with n,
                    neither the age rule nor the free-space rule removing n, r_m > 0, r_n > 0,
                    dot = (nm.x nn.x + nm.y nn.y) + nm.z nn.z > dot_th, and with d = p_n - p_m,
                    d2 = (d.x d.x + d.y d.y) + d.z d.z <= (r_m + r_n)^2
    winner          the candidate of smallest (d2, n)
    absorb          c = c_m + c_n, inv = 1 / c (1 / 1 for c = 0); position, normal, colour and radius of m become
                    ((c_m x_m) + (c_n x_n)) * inv, its ccount c; n joins the step's removals
    pruned step s   one stable removal of the age rule's rows, the violators and the absorbed rows (free_space_oracle)

Every decision is taken on the map the fusion left, before any absorption, under no_grad; the absorption itself is
separate float32 torch ops, so the oracle's autograd gives its gradient."""
import math

import torch

import free_space_oracle as fo
import gsx_oracle as oracle
import prune_oracle as po
import radii_oracle as ro

F32 = torch.float32


def age_removals(pm, c_stable, t_max):
    """Per element, bool (N_b,): the rows the age rule removes in the pruned step pm.step (before prune_step stamps
    the rows it has not seen yet with that step)."""
    m, s = pm.smap, pm.step
    out = []
    for b in range(m.B):
        count = m.points[b].shape[0]
        known = 0 if pm.created is None else pm.created[b].shape[0]
        created = torch.full((count,), s, dtype=torch.int64)
        if known:
            created[:known] = pm.created[b]
        remove = torch.zeros(count, dtype=torch.bool)
        if s >= t_max:
            remove = (created == s - t_max) & (m.ccounts[b][:, 0] < torch.tensor(c_stable, dtype=F32))
        out.append(remove)
    return out


def merge_pairs(smap, radii, table, pose, K, H, W, c_stable, dot_th, removed):
    """Per element, the absorbed pairs as an int64 (A, 2) tensor of rows [m, n], in pixel order.  smap / radii: the map
    after the fusion whose unique correspondence table is `table` (rows [b, n, h, w]); removed[b]: bool (N_b,), the rows
    the age and free-space rules remove in this step."""
    out = [torch.empty((0, 2), dtype=torch.int64) for _ in range(smap.B)]
    if not smap.has_points or table.shape[0] == 0:
        return out
    with torch.no_grad():
        pts, nrm, _, cc = smap.padded()
        active = oracle.find_active_map_points(smap, pose, K, H, W)
        for i in range(smap.B):
            tb = table[table[:, 0] == i]
            if tb.shape[0] == 0:
                continue
            count = smap.points[i].shape[0]
            target = torch.zeros(count, dtype=torch.bool)
            target[tb[:, 1]] = True
            absorber = torch.full((H, W), -1, dtype=torch.int64)
            m_all, h_all, w_all = tb[:, 1], tb[:, 2], tb[:, 3]
            ok = (cc[i, m_all, 0] >= torch.tensor(c_stable, dtype=F32)) & ~removed[i][m_all]
            absorber[h_all[ok], w_all[ok]] = m_all[ok]
            act = active[active[:, 0] == i]
            n, h, w = act[:, 1], act[:, 2], act[:, 3]
            m = absorber[h, w]
            keep = (m >= 0) & (n != m) & ~target[n] & ~removed[i][n]
            n, h, w, m = n[keep], h[keep], w[keep], m[keep]
            r = radii[i][:, 0]
            rm, rn = r[m], r[n]
            nm, nn = nrm[i, m], nrm[i, n]
            dot = (nm[:, 0] * nn[:, 0] + nm[:, 1] * nn[:, 1]) + nm[:, 2] * nn[:, 2]
            d = pts[i, n] - pts[i, m]
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            rr = rm + rn
            cand = (rm > 0) & (rn > 0) & (dot > torch.tensor(dot_th, dtype=F32)) & (d2 <= rr * rr)
            n, h, w, m, d2 = n[cand], h[cand], w[cand], m[cand], d2[cand]
            if n.numel() == 0:
                continue
            # smallest (d2, n) per pixel: sort by n, then stably by d2, then stably by pixel; the first of each pixel
            pix = h * W + w
            o = torch.argsort(n, stable=True)
            o = o[torch.argsort(d2[o], stable=True)]
            o = o[torch.argsort(pix[o], stable=True)]
            first = torch.ones(o.numel(), dtype=torch.bool)
            first[1:] = pix[o][1:] != pix[o][:-1]
            o = o[first]
            out[i] = torch.stack([m[o], n[o]], 1)
    return out


def absorb(smap, radii, pairs):
    """The absorptions of `pairs` (merge_pairs), out of place: returns (SurfelMap, radii) whose rows m are the
    confidence-weighted means; rows n are still there (the pruned step removes them)."""
    pts, nrm, col, cc, rad = [], [], [], [], []
    for i in range(smap.B):
        P, N, C, Q, R = (t[i].clone() for t in (smap.points, smap.normals, smap.colors, smap.ccounts, radii))
        if pairs[i].shape[0]:
            m, n = pairs[i][:, 0], pairs[i][:, 1]
            cm, cn = smap.ccounts[i][m], smap.ccounts[i][n]
            tot = cm + cn
            inv = 1 / torch.where(tot == 0, torch.ones_like(tot), tot)
            mix = lambda x: ((cm * x[m]) + (cn * x[n])) * inv
            P[m], N[m], C[m] = mix(smap.points[i]), mix(smap.normals[i]), mix(smap.colors[i])
            R[m] = mix(radii[i])
            Q[m] = tot
        pts.append(P), nrm.append(N), col.append(C), cc.append(Q), rad.append(R)
    return oracle.SurfelMap(pts, nrm, col, cc), rad


def run_pointfusion(rgb, depth, K, poses=None, *, c_stable, t_max, margin=None, merge=True, odom="gt", dist_th=0.05,
                    angle_th=20.0, sigma=0.6, dsratio=4, numiters=20, damp=1e-8, dist_thresh=None, lambda_max=2.0,
                    B=1.0, B2=1.0, nu=200.0, association="nn", pm=None, radii=None, s_begin=0, ring=None):
    """free_space_oracle.run_pointfusion with surfel radii and, with merge, the merging of overlapping surfels in every
    pruned step (margin None: no free-space violator, as margin = inf).  pm / radii continue an earlier run from frame
    s_begin.  ring: a free_space_oracle.PositionalRingPruner replayed on the same removals.  Returns
    (PrunedMap, radii per element (N_b, 1), poses (B,L,4,4), rows absorbed per element)."""
    Bn, L, H, W, _ = depth.shape
    dot_th = math.cos(angle_th * math.pi / 180)
    kw = dict(numiters=numiters, damp=damp, dist_thresh=dist_thresh)
    if odom == "gradicp":
        kw.update(lambda_max=lambda_max, B=B, B2=B2, nu=nu)
    pm = po.PrunedMap() if pm is None else pm
    out_poses = torch.empty(Bn, L, 4, 4)
    absorbed = [0] * Bn
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
        radii = ro.fuse_radii(pm.smap, radii, maps, d, K, table, sigma)
        pm.smap = oracle.fuse_with_map(pm.smap, maps, c, table, sigma)
        if pm.smap.has_points:
            pz = pose.detach()
            if margin is not None:
                bound = fo.bound_image(pm.smap, table, pz, K4, H, W, c_stable)
                viol = fo.violators(pm.smap, bound, pz, K4, margin)
            else:
                viol = [torch.zeros(n, dtype=torch.bool) for n in pm.smap.counts()]
            extra = viol
            if merge:
                removed = [a | v for a, v in zip(age_removals(pm, c_stable, t_max), viol)]
                pairs = merge_pairs(pm.smap, radii, table, pz, K4, H, W, c_stable, dot_th, removed)
                pm.smap, radii = absorb(pm.smap, radii, pairs)
                extra = []
                for i, v in enumerate(viol):
                    v = v.clone()
                    v[pairs[i][:, 1]] = True
                    extra.append(v)
                    absorbed[i] += int(pairs[i].shape[0])
            if ring is not None:
                ring(pm.smap.clone(), c_stable, extra)
            keeps = fo.prune_step(pm, c_stable, t_max, extra)
            radii = [r[k] for r, k in zip(radii, keeps)]
        else:
            pm.step += 1
            if ring is not None:
                ring.step += 1
        prev_pose = pose
        out_poses[:, s] = pose
    return pm, radii, out_poses, absorbed
