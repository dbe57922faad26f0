"""Oracle of the mocap driver (renderih_b200/mocap_optimize.py, csrc/scene.cu).

frame_geometry / search_anchors restate update_scene's geometry (batch_optimize_mocap_origin.py:256-270) and search_anchors (:62-130) in
numpy, one frame at a time, with the port's tie rule (equal distances go to the lowest index: a stable sort) and its left-to-right float32
dot product; every other operation is numpy's, in numpy's order, so on the same vertices the kernel must agree exactly on every decision.
scene_frames() runs them over a batch and also returns each frame's margins: how close a distance came to its threshold or to the next
candidate, and a normal dot product to -0.6.

eager_optimize_mocap() is the reference's driver loop (main, :373-593, discrete path) one frame at a time: per frame, two batch-1 CUDA
ManoLayer forwards copied to the host, the numpy geometry and search above, the frames stacked as combine_frame_inf does, then run_sample's
host-to-device copies and GeOptimizer.set_opt_val / optimize.  It is the GPU tests' oracle and the benchmark's baseline; translations are
held in float32, as the port holds them.
"""
import time

import numpy as np
import torch

DIM = 4
D_FRESH, D_PREV, AGAINST = 0.015, 0.02, np.float32(-0.6)


def frame_geometry(verts, tsl, fvi, aw):
    """One hand of one frame: centred vertices [778,3] float32 + translation [3] float32 -> (anchors [A,3] float64, normals [A,3] float32,
    not negated)."""
    v = (np.asarray(verts, np.float32) + np.asarray(tsl, np.float32))[fvi]          # [A,3,3]
    e1, e2 = v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]
    anchors = (aw[:, 0:1] * e1 + aw[:, 1:2] * e2) + v[:, 0]
    n = np.cross(e1, e2)
    n = n / np.linalg.norm(n, axis=-1)[:, np.newaxis]
    return anchors, n


def dots(sub_normals, main_normals):
    """[A,A] float32 sub_i . main_j, summed left to right."""
    s, m = sub_normals[:, np.newaxis, :], main_normals[np.newaxis, :, :]
    return (s[..., 0] * m[..., 0] + s[..., 1] * m[..., 1]) + s[..., 2] * m[..., 2]


def search_anchors(main_anchors, sub_anchors, main_normals, sub_normals, class_types, prev_anchor_id=None):
    """search_anchors (:62-130) -> (vertex_contact [A] int64, anchor_id [A,4] int64, anchor_elasti [A,4] float32, anchor_padding_mask
    [A,4] int64, margin_d, margin_dot): margin_d is the smallest |d - threshold| and gap between the 4th and 5th smallest distances
    (unless the 5th is the masked 1000.0) over the anchors, in metres; margin_dot the smallest |dot + 0.6| (fresh branch)."""
    A = sub_anchors.shape[0]
    anchor_id = np.zeros([A, DIM], dtype=np.int64)
    vertex_contact = np.zeros(A, dtype=np.int64)
    elasti = np.zeros([A, DIM], dtype=np.float32)
    pad = np.zeros([A, DIM], dtype=np.int64)
    margin, margin_dot = np.inf, np.inf
    if prev_anchor_id is None:
        dot = dots(sub_normals, main_normals)
        margin_dot = float(np.abs(dot.astype(np.float64) + 0.6).min())
    for i in range(A):
        dis = np.linalg.norm(sub_anchors[i] - main_anchors, axis=-1)
        if prev_anchor_id is not None:
            t = D_PREV
            d = 1000 * np.ones(dis.shape, dtype=dis.dtype)
            d[prev_anchor_id[i]] = dis[prev_anchor_id[i]]
            dis = d
            ids = np.asarray(prev_anchor_id[i], dtype=np.int64)
        else:
            t = D_FRESH
            dis[dot[i] > AGAINST] = 1000.0
            order = np.argsort(dis, kind='stable')
            ids = order[:DIM]
            if dis[order[DIM]] != 1000.0:
                margin = min(margin, float(dis[order[DIM]] - dis[order[DIM - 1]]))
        contact_able = dis < t
        k = contact_able * (0.5 * np.cos(np.pi * dis / t) + 0.5)
        real = dis[dis != 1000.0]
        if real.size:
            margin = min(margin, float(np.abs(real - t).min()))
        vertex_contact[i] = contact_able.sum() > 0
        anchor_id[i] = ids
        elasti[i] = k[ids]
        pad[i] = elasti[i] > 0.0
    elasti[(class_types.repeat(DIM).reshape([-1, DIM]) != 4) * (class_types[anchor_id] != 4)] *= 0.3
    return vertex_contact, anchor_id, elasti, pad, margin, margin_dot


def scene_frames(v_main, v_sub, t_main, t_sub, fvi, aw, class_types, prev=None):
    """update_scene's search over B frames from centred vertices [B,778,3] and translations [B,3] (float32 arrays) -> dict of stacked
    arrays: vertex_contact, anchor_id, anchor_elasti, anchor_padding_mask, optimize_it [B,1] bool, obj_anchors / obj_normals float32,
    margin / margin_dot [B]."""
    out = {k: [] for k in ('vertex_contact', 'anchor_id', 'anchor_elasti', 'anchor_padding_mask', 'optimize_it', 'obj_anchors',
                           'obj_normals', 'margin', 'margin_dot')}
    for b in range(len(v_main)):
        ma, mn = frame_geometry(v_main[b], t_main[b], fvi, aw)
        sa, sn = frame_geometry(v_sub[b], t_sub[b], fvi, aw)
        sn = -sn
        vc, ids, el, pad, margin, margin_dot = search_anchors(ma, sa, mn, sn, class_types, None if prev is None else prev[b])
        for k, v in (('vertex_contact', vc), ('anchor_id', ids), ('anchor_elasti', el), ('anchor_padding_mask', pad),
                     ('optimize_it', np.asarray([vc.sum() > 0])), ('obj_anchors', sa.astype(np.float32)), ('obj_normals', sn),
                     ('margin', margin), ('margin_dot', margin_dot)):
            out[k].append(v)
    return {k: np.stack(v) if not k.startswith('margin') else np.asarray(v) for k, v in out.items()}


def tables(scene):
    """(fvi [A,3] int64, aw [A,2] float64, class types [A] int64) of a renderih_b200 Scene, on the host."""
    return scene._fvi.cpu().numpy().astype(np.int64), scene._aw.cpu().numpy(), scene._cls.cpu().numpy().astype(np.int64)


def eager_optimize_mocap(raw_data, hoptim, scene, batch_size, optimize_interval=1, mocap_scale=1.0, timing=None):
    """main's discrete path (:373-593) with the reference's per-frame loop structure (see the module docstring) -> the dict main saves.
    timing, if a dict, receives 'scene_s' (per-frame preparation, host clock) and 'optim_s' (run_sample)."""
    from renderih_b200 import mocap_optimize as MO
    dev = scene.device
    fvi, aw, cls = tables(scene)
    frames = np.arange(0, len(raw_data['right']['rot']), optimize_interval)
    quat = {s: MO.euler_to_mano_quat(np.asarray(raw_data[s]['rot'])[frames], s, *scene.converter[s]) for s in ('right', 'left')}
    tsl = {s: (np.asarray(raw_data[s]['loc'])[frames] / 100 * mocap_scale).astype(np.float32) for s in ('right', 'left')}
    shape = torch.cat([torch.from_numpy(np.asarray(raw_data[s]['shape']).astype(np.float32)).squeeze(1) for s in ('right', 'left')], 1)
    n = len(frames)
    t_scene = t_opt = 0.0

    def frame(f, prev):
        shp = shape[f:f + 1].to(dev)
        with torch.no_grad():
            vm = scene.main_hand(torch.from_numpy(quat['right'][f:f + 1]).to(dev), shp[:, :10])[0][0].cpu().numpy()
            vs = scene.sub_hand(torch.from_numpy(quat['left'][f:f + 1]).to(dev), shp[:, 10:])[0][0].cpu().numpy()
        r = scene_frames(vm[None], vs[None], tsl['right'][f:f + 1], tsl['left'][f:f + 1], fvi, aw, cls, None if prev is None else prev[None])
        return {k: v[0] for k, v in r.items()}

    base = (hoptim.coef_val['lambda_repulsion_loss'], hoptim.coef_val['lambda_contact_loss'])
    ids = None
    for rep, con, n_iter, recompute in MO.attempt_table(*base):
        hoptim.coef_val['lambda_repulsion_loss'] = rep
        hoptim.coef_val['lambda_contact_loss'] = con
        hoptim.n_iter = n_iter
        t0 = time.perf_counter()
        if recompute:
            ids = np.asarray([frame(f, None)['anchor_id'] for f in range(n)])
        t_scene += time.perf_counter() - t0
        for s in range(0, n, batch_size):
            e = min(s + batch_size, n)
            t0 = time.perf_counter()
            fr = [frame(f, ids[f]) for f in range(s, e)]
            info = {k: np.stack([x[k] for x in fr]) for k in fr[0] if not k.startswith('margin')}
            t1 = time.perf_counter()
            to = lambda a, dt: torch.from_numpy(np.asarray(a)).to(dt).to(dev)
            hp, op = to(quat['right'][s:e], torch.float32), to(quat['left'][s:e], torch.float32)
            zeros = torch.zeros(e - s, 16, device=dev)
            hoptim.set_opt_val(vertex_contact=to(info['vertex_contact'], torch.long), contact_region=to(np.zeros_like(info['vertex_contact']), torch.long),
                               anchor_id=to(info['anchor_id'], torch.long), anchor_elasti=to(info['anchor_elasti'], torch.float32),
                               anchor_padding_mask=to(info['anchor_padding_mask'], torch.long), hand_shape_init=shape[s:e].to(dev),
                               hand_tsl_init=to(tsl['right'][s:e], torch.float32), hand_pose_gt=([0], hp[:, 0:1, :]),
                               hand_pose_init=(list(range(1, 16)), hp[:, 1:, :]), runtime_vis=9527,
                               obj_tsl_init=to(tsl['left'][s:e], torch.float32), obj_pose_gt=([0], op[:, 0:1, :]),
                               obj_pose_init=(list(range(1, 16)), op[:, 1:, :]), obj_anchors=to(info['obj_anchors'], torch.float32),
                               obj_normals=to(info['obj_normals'], torch.float32), optimize_it=to(info['optimize_it'], torch.bool),
                               batch_size=e - s, consistent_mask=[zeros, zeros])
            res = hoptim.optimize(progress=False)
            t_scene += t1 - t0
            t_opt += time.perf_counter() - t1
            quat['right'][s:e] = res['optimized_hand_pose'].numpy()
            tsl['right'][s:e] = res['optimized_hand_tsl'].numpy()
            quat['left'][s:e] = res['optimized_sub_hand_pose'].numpy()
            tsl['left'][s:e] = res['optimized_sub_hand_tsl'].numpy()
    if timing is not None:
        timing.update(scene_s=t_scene, optim_s=t_opt)
    out = {k: (dict(v) if isinstance(v, dict) else v) for k, v in raw_data.items()}
    for side, cols in (('right', slice(0, 10)), ('left', slice(10, None))):
        out[side]['rot'] = MO.mano_quat_to_euler(quat[side], side, *scene.converter[side])
        out[side]['loc'] = tsl[side].astype(np.float64) * 100
        out[side]['shape'] = shape.numpy()[:, cols]
    return out


def synthetic_mocap(n_frames, seed, spread=0.035, joint_deg=15.0, root_deg=40.0):
    """A mocap dict {'right'/'left': {'rot' [N,16,3] euler degrees, 'loc' [N,3] centimetres, 'shape' [N,1,10]}}: both hands near one
    another, so that some frames are in contact and some are not; joint and root angles are normal with the given deviations."""
    rng = np.random.default_rng(seed)
    d = {}
    for side, x in (('right', 1.0), ('left', -1.0)):
        rot = rng.normal(size=(n_frames, 16, 3)) * joint_deg
        rot[:, 0] = rng.normal(size=(n_frames, 3)) * root_deg
        loc = np.tile([[x * 2.0, 0.0, 0.0]], (n_frames, 1)) + rng.normal(size=(n_frames, 3)) * spread * 100
        d[side] = {'rot': rot, 'loc': loc, 'shape': rng.normal(size=(n_frames, 1, 10)) * 0.5}
    return d
