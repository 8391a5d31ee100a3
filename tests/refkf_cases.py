"""Tracking::TrackReferenceKeyFrame + TrackLocalMap (src/Tracking.cc:796-838, :969-1000 with SearchLocalPoints :1262-1312) composed from the CPU oracle's
functions -- the checker of sgs_tracker_refkf_chain_device (tests/test_gpu_refkf_chain.py), itself pinned against the reference's own tracking code in
tests/test_refkf_chain_ref.py -- and a vocabulary trained on the frames' descriptors."""
import numpy as np

import oracle as O


def train_vocabulary(desc, k, L, seed=0, rounds=3):
    """A DBoW2-shaped tree trained on `desc` [N][32] by hierarchical k-medians in Hamming space (k children per inner node, every leaf at level L, the
    children of a node numbered consecutively as TemplatedVocabulary::HKmeansStep creates them).  Leaf weights: log(N / n_i) over the training features
    (n_i = features filed under leaf i; a leaf that none reaches gets log N)."""
    rng = np.random.RandomState(seed)
    bits = np.unpackbits(np.ascontiguousarray(desc, np.uint8), axis=1)
    parent, nodes, level = [-1], [np.zeros(256, np.uint8)], [0]
    members = {0: np.arange(len(bits))}
    queue = [0]
    while queue:
        nid = queue.pop(0)
        if level[nid] == L:
            continue
        idx = members[nid]
        if len(idx) == 0:
            cent = [nodes[nid] ^ (rng.rand(256) < 0.1).astype(np.uint8) for _ in range(k)]
            assign = np.zeros(0, np.int64)
        else:
            cent = [bits[idx[j]] for j in rng.choice(len(idx), k, replace=len(idx) < k)]
            for _ in range(rounds):
                d = (bits[idx][:, None, :] != np.stack(cent)[None]).sum(2)
                assign = d.argmin(1)
                cent = [((bits[idx[assign == c]].sum(0) * 2) > (assign == c).sum()).astype(np.uint8) if (assign == c).any() else cent[c] for c in range(k)]
            d = (bits[idx][:, None, :] != np.stack(cent)[None]).sum(2)
            assign = d.argmin(1)
        for c in range(k):
            cid = len(parent)
            parent.append(nid); nodes.append(cent[c]); level.append(level[nid] + 1)
            members[cid] = idx[assign == c] if len(idx) else idx
            queue.append(cid)
    parent = np.array(parent, np.int32); level = np.array(level)
    weight = np.zeros(len(parent), np.float64)
    for i in np.nonzero(level == L)[0]:
        weight[i] = np.log(len(bits) / max(len(members[i]), 1))
    return dict(k=k, L=L, parent=parent, desc=np.packbits(np.stack(nodes), axis=1), weight=weight)


def oracle_refkf(cur, V, kf, Tlast, lm, seen_in, camd, camv, sf, isig, th_local, pc, tcw_first=None):
    """One frame of the chain.  cur: O.FrameArrays of the frame; V: O.Vocabulary; kf: the reference key frame (desc, angle, xyz, flags, lid, n); lm: the
    local map (bench.make_local_map); seen_in: [len(lm['valid'])] points already seen in the frame, or None.  tcw_first: run the local half from this pose
    instead of the oracle's own first pose.  Returns stats [8] and, for a frame past the 15-match gate, both poses, the matches after the discard (mp1),
    the final ids (mp) and outlier flags."""
    st = np.zeros(8, np.int64)
    m = int(kf['n'])
    fl = kf['flags'][:m]
    _, fw, fnode = V.transform(cur.desc, 4)
    _, kw, knode = V.transform(kf['desc'][:m], 4)
    valid = ((fl & 1) != 0) & ((fl & 4) == 0)
    nm, mf = O.search_by_bow(knode, kw, valid.astype(np.uint8), kf['desc'][:m], kf['angle'][:m], fnode, fw, cur.desc, cur.keysUn['angle'], 0.7, True)
    st[0] = nm
    if nm < 15:
        return dict(stats=st)
    st[1] = 1
    N = cur.c.N
    mp = np.asarray(mf, np.int64).copy()
    kxy = np.stack([cur.keysUn['x'], cur.keysUn['y']], 1)
    po = lambda T, has, xyz: O.pose_optimization(T, has, xyz, kxy, cur.keysUn['octave'], cur.uRight, isig, camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'])
    xyz = np.zeros((N, 3), np.float32); xyz[mp >= 0] = kf['xyz'][mp[mp >= 0]]
    _, T1, out1 = po(Tlast, (mp >= 0).astype(np.uint8), xyz)
    seen = np.zeros(len(lm['valid']), np.uint8) if seen_in is None else np.asarray(seen_in, np.uint8).copy()
    obs = np.zeros(N, np.uint8)
    nmatches, nmap = nm, 0
    for i in range(N):
        if mp[i] >= 0:
            lid = kf['lid'][mp[i]] if kf['lid'] is not None else -1
            if lid >= 0: seen[lid] = 1
            if out1[i]:
                mp[i] = -1; nmatches -= 1
            else:
                if fl[mp[i]] & 2: nmap += 1
                if fl[mp[i]] & 4: mp[i] = -1
                else: obs[i] = (fl[mp[i]] >> 1) & 1
    st[3] = nmatches; st[4] = nmap
    mp1 = mp.copy()
    T1u = T1 if tcw_first is None else np.asarray(tcw_first, np.float32).reshape(4, 4)
    n = lm['n']
    fr = O.is_in_frustum(T1u, camv, 8, float(O.logf(sf[1])), lm['xyz'][:n], lm['nrm'][:n], lm['mn'][:n], lm['mx'][:n], 0.5)
    inview = fr['inview'] & lm['valid'][:n] & (1 - seen[:n])
    st[5] = int(inview.sum())
    nml, mp2, obs2, _ = O.search_by_projection_local(cur, inview, fr['proj_x'], fr['proj_y'], fr['proj_xr'], fr['level'], fr['view_cos'], lm['dsc'][:n], lm['obs'][:n],
                                                     th_local, 0.8, mp, obs, id_base=pc)
    st[6] = nml
    xyz2 = np.zeros((N, 3), np.float32)
    a = (mp2 >= 0) & (mp2 < pc); b = mp2 >= pc
    xyz2[a] = kf['xyz'][mp2[a]]; xyz2[b] = lm['xyz'][mp2[b] - pc]
    has2 = (mp2 >= 0).astype(np.uint8)
    _, T2, out2 = po(T1u, has2, xyz2)
    out2 = out2 & has2
    st[7] = int(((mp2 >= 0) & (out2 == 0) & (obs2 != 0)).sum())
    return dict(stats=st, T1=T1, T2=T2, mp1=mp1, mp=mp2, outlier=out2)


def motion_discards(cur, mp_track, nm_track, ti, f, lm, camd, isig, th):
    """Local-map ids of the outliers TrackWithMotionModel's discard drops (src/Tracking.cc:940-957), for a frame whose matches after the wide-window retry
    reach 20 (none otherwise: :933 returns first)."""
    m = int(ti['ln'][f]); fl = ti['lflags'][f, :m]
    Tc = ti['Tc'][f].reshape(4, 4); Tl = ti['T'][f].reshape(4, 4)
    mp, nm = mp_track.copy(), nm_track
    if nm < 20:
        nm, mp, _ = O.search_by_projection_last(cur, Tc, Tl, fl & 1, ti['lxyz'][f, :m], ti['ldesc'][f, :m], (fl >> 1) & 1, ti['loct'][f, :m], ti['lang'][f, :m], 2 * th)
    out = np.zeros(len(lm['valid']), np.uint8)
    if nm < 20:
        return out
    N = cur.c.N
    xyz = np.zeros((N, 3), np.float32); xyz[mp >= 0] = ti['lxyz'][f, mp[mp >= 0]]
    kxy = np.stack([cur.keysUn['x'], cur.keysUn['y']], 1)
    _, _, out1 = O.pose_optimization(Tc, (mp >= 0).astype(np.uint8), xyz, kxy, cur.keysUn['octave'], cur.uRight, isig, camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'])
    for i in np.nonzero((mp >= 0) & (out1 != 0))[0]:
        lid = lm['lid'][mp[i]]
        if lid >= 0: out[lid] = 1
    return out
