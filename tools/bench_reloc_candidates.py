"""Times KeyFrameDatabase::DetectRelocalizationCandidates on the device (sgs_kfdb_reloc_candidates_device) with CUDA events, and the Python
restatement of tests/kfdb_cases.py on the CPU for the same queries:
  - 64 rows, one per map, against 64 maps of 1024 key frames each (a batch of lost streams);
  - one row against one map of 8192 key frames.
BowVectors are random: about 700 words per frame and key frame out of a 20000-word vocabulary (ORBvoc has 10^6 words, but a relocalising frame
shares far more words with its map than uniform draws from 10^6 would), values L1-normalised.  Prints one JSON line with the card's name and power
limit read in the same run.  A second JSON line times KeyFrameDatabase::DetectLoopCandidates with DetectLoop's minScore
(sgs_kfdb_loop_candidates_device) on the same maps, right after the relocalisation leg: each row a new key frame near a key frame of its map,
built like the relocalising frames, with the 30 slots that follow that key frame in its map as its connected set and BowVectors near the first 20
of them as its covisible key frames.  Needs a CUDA device."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, 'sg-slam_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)

import kfdb_cases as K  # noqa: E402
import kfdb_loop_cases as KL  # noqa: E402
from pysgs import binding as B  # noqa: E402


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).splitlines()[0]
        name, power = [x.strip() for x in out.split(',')]
        return name, power
    except Exception as e:      # the timing still stands; the card is named by torch
        import torch
        return torch.cuda.get_device_name(0), 'unknown (%s)' % type(e).__name__


def rows(bows, cap):
    """BowVectors as [n][cap] word and value rows and their lengths"""
    w = np.zeros((len(bows), cap), np.int32); v = np.zeros((len(bows), cap)); n = np.zeros(len(bows), np.int32)
    for i, (ids, vals) in enumerate(bows):
        w[i, :len(ids)] = ids; v[i, :len(ids)] = vals; n[i] = len(ids)
    return w, v, n


def near(rng, ids, nvoc):
    """a BowVector near the one with words ids: a third of them replaced, new values, L1-normalised"""
    keep = ids[rng.uniform(size=len(ids)) > 0.33]
    new = np.setdiff1d(rng.choice(nvoc, len(ids) - len(keep), replace=False), keep)
    return K.normalized(np.concatenate([keep, new]), rng.uniform(0.05, 1.0, len(keep) + len(new)))


def timed(call, iters):
    """CUDA-event ms per call over iters calls, after 20 warm-up calls"""
    import torch
    for _ in range(20):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


class Maps:
    """nmaps maps of per_map random key frames in one database, ten same-map neighbours per key frame"""

    def __init__(self, nmaps, per_map, nvoc, nwords, rng):
        import torch
        self.nmaps, self.per_map, self.nvoc, self.K = nmaps, per_map, nvoc, nmaps * per_map
        self.cap = nwords + 64
        self.L = B.lib()
        self.db = C.c_void_p()
        B.check(self.L.sgs_kfdb_create(0, nmaps, self.K, self.cap, C.byref(self.db)))
        self.bows = [K.random_bow(rng, nvoc, nwords - 50, nwords + 50) for _ in range(self.K)]
        w, v, n = rows(self.bows, self.cap)
        slots = np.arange(self.K, dtype=np.int32); self.maps = (slots // per_map).astype(np.int32)
        dw, dv, dn = torch.from_numpy(w).cuda(), torch.from_numpy(v).cuda(), torch.from_numpy(n).cuda()
        B.check(self.L.sgs_kfdb_add(self.db, self.K, B._p(slots), B._p(self.maps), dw.data_ptr(), dv.data_ptr(), dn.data_ptr(), self.cap, None))
        self.covis = np.full((self.K, 10), -1, np.int32)
        for s in range(self.K):
            self.covis[s] = self.following(s, 10)
        self.dcov = torch.from_numpy(self.covis).cuda()

    def following(self, s, k):
        """the k slots after slot s in its map, cyclically"""
        base = (s // self.per_map) * self.per_map
        return (base + (s - base + np.arange(1, k + 1)) % self.per_map).astype(np.int32)

    def close(self):
        self.L.sgs_kfdb_destroy(self.db)


def case(M, iters, cpu_rows, rng):
    """the relocalisation leg: each row a key frame of its map with a third of its words replaced (a frame near that key frame)"""
    import torch
    L, F, cap, nvoc = M.L, M.nmaps, M.cap, M.nvoc
    qb = [near(rng, M.bows[f * M.per_map + int(rng.integers(M.per_map))][0], nvoc) for f in range(F)]
    dq = [torch.from_numpy(x).cuda() for x in rows(qb, cap)]
    cc = 64
    cand = torch.zeros((F, cc), dtype=torch.int32, device='cuda'); nc = torch.zeros(F, dtype=torch.int32, device='cuda')
    st = torch.zeros((F, 4), dtype=torch.int32, device='cuda')
    qm = np.arange(F, dtype=np.int32)
    s = torch.cuda.current_stream().cuda_stream

    def call():
        B.check(L.sgs_kfdb_reloc_candidates_device(M.db, F, B._p(qm), dq[0].data_ptr(), dq[1].data_ptr(), dq[2].data_ptr(), cap, M.dcov.data_ptr(),
                                                   cand.data_ptr(), cc, nc.data_ptr(), st.data_ptr(), C.c_void_p(s)))
    ms = timed(call, iters)
    # the restatement on the CPU, the same queries (rows up to cpu_rows), checked against the device's last call
    ref = K.Database(M.K)
    for i in range(M.K):
        ref.add(i, int(M.maps[i]), *M.bows[i])
    ncpu = min(F, cpu_rows)
    t0 = time.perf_counter()
    want = [ref.query(f, *qb[f], M.covis, cc) for f in range(ncpu)]
    cpu_ms = (time.perf_counter() - t0) * 1e3 * F / ncpu
    got_c, got_n, got_s = cand.cpu().numpy(), nc.cpu().numpy(), st.cpu().numpy()
    same = all(list(got_s[f]) == want[f][1] and list(got_c[f, :got_n[f]]) == want[f][0][:cc] for f in range(ncpu))
    return dict(rows=F, keyframes_per_map=M.per_map, words=M.cap - 64, device_ms_per_call=round(ms, 4), restatement_cpu_ms_per_call=round(cpu_ms, 1),
                cpu_rows_timed=ncpu, equal_to_restatement=bool(same), mean_sharing=float(got_s[:, 0].mean()), mean_scored=float(got_s[:, 2].mean()))


def loop_case(M, iters, cpu_rows, rng, nconn=30, ncov=20):
    """the loop leg on the same maps: each row a new key frame near key frame c of its map, connected to the nconn slots after c, with BowVectors
    near the first ncov of them as its covisible key frames"""
    import torch
    L, F, cap, nvoc = M.L, M.nmaps, M.cap, M.nvoc
    qb, conns, covs = [], [], []
    for f in range(F):
        c = f * M.per_map + int(rng.integers(M.per_map))
        qb.append(near(rng, M.bows[c][0], nvoc))
        conns.append(M.following(c, nconn))
        covs.append([near(rng, M.bows[int(s)][0], nvoc) for s in conns[-1][:ncov]])
    conn_off = np.arange(0, F * nconn + 1, nconn, dtype=np.int32); cov_off = np.arange(0, F * ncov + 1, ncov, dtype=np.int32)
    dq = [torch.from_numpy(x).cuda() for x in rows(qb, cap)]
    dc = [torch.from_numpy(x).cuda() for x in rows([b for cs in covs for b in cs], cap)]
    dconn = torch.from_numpy(np.concatenate(conns)).cuda()
    cc = 64
    cand = torch.zeros((F, cc), dtype=torch.int32, device='cuda'); nc = torch.zeros(F, dtype=torch.int32, device='cuda')
    st = torch.zeros((F, 4), dtype=torch.int32, device='cuda'); mn = torch.zeros(F, dtype=torch.float32, device='cuda')
    qm = np.arange(F, dtype=np.int32)
    s = torch.cuda.current_stream().cuda_stream

    def call():
        B.check(L.sgs_kfdb_loop_candidates_device(M.db, F, B._p(qm), dq[0].data_ptr(), dq[1].data_ptr(), dq[2].data_ptr(), cap, B._p(conn_off),
                                                  dconn.data_ptr(), B._p(cov_off), dc[0].data_ptr(), dc[1].data_ptr(), dc[2].data_ptr(),
                                                  M.dcov.data_ptr(), cand.data_ptr(), cc, nc.data_ptr(), st.data_ptr(), mn.data_ptr(), C.c_void_p(s)))
    ms = timed(call, iters)
    ref = KL.LoopDatabase(M.K)
    for i in range(M.K):
        ref.add(i, int(M.maps[i]), *M.bows[i])
    ncpu = min(F, cpu_rows)
    want = [ref.loop(f, *qb[f], conns[f].tolist(), covs[f], M.covis, -1, cc) for f in range(ncpu)]
    got_c, got_n, got_s, got_m = cand.cpu().numpy(), nc.cpu().numpy(), st.cpu().numpy(), mn.cpu().numpy()
    same = all(list(got_s[f]) == want[f][1] and list(got_c[f, :got_n[f]]) == want[f][0][:cc] and got_m[f].tobytes() == np.float32(want[f][2]).tobytes()
               for f in range(ncpu))
    return dict(rows=F, keyframes_per_map=M.per_map, words=cap - 64, connected=nconn, covisible=ncov, device_ms_per_call=round(ms, 4),
                rows_checked=ncpu, equal_to_restatement=bool(same), mean_sharing=float(got_s[:, 0].mean()), mean_scored=float(got_s[:, 2].mean()),
                mean_candidates=float(got_n.mean()))


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--cpu-rows', type=int, default=8)
    a = ap.parse_args()
    name, power = card()
    reloc, loop = [], []
    for nmaps, per_map, cpu_rows, seed in ((64, 1024, a.cpu_rows, 1), (1, 8192, 1, 2)):
        rng = np.random.default_rng(seed)
        M = Maps(nmaps, per_map, 20000, 700, rng)
        reloc.append(case(M, a.iters, cpu_rows, rng))
        loop.append(loop_case(M, a.iters, cpu_rows, rng))
        M.close()
    print(json.dumps(dict(card=name, power_limit=power, cases=reloc)))
    print(json.dumps(dict(query='loop', card=name, power_limit=power, cases=loop)))
