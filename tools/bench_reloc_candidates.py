"""Times KeyFrameDatabase::DetectRelocalizationCandidates on the device (sgs_kfdb_reloc_candidates_device) with CUDA events, and the Python
restatement of tests/kfdb_cases.py on the CPU for the same queries:
  - 64 rows, one per map, against 64 maps of 1024 key frames each (a batch of lost streams);
  - one row against one map of 8192 key frames.
BowVectors are random: about 700 words per frame and key frame out of a 20000-word vocabulary (ORBvoc has 10^6 words, but a relocalising frame
shares far more words with its map than uniform draws from 10^6 would), values L1-normalised.  Prints one JSON line with the card's name and power
limit read in the same run.  Needs a CUDA device."""
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
from pysgs import binding as B  # noqa: E402


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).splitlines()[0]
        name, power = [x.strip() for x in out.split(',')]
        return name, power
    except Exception as e:      # the timing still stands; the card is named by torch
        import torch
        return torch.cuda.get_device_name(0), 'unknown (%s)' % type(e).__name__


def case(nmaps, per_map, nvoc, nwords, iters, cpu_rows, seed):
    import torch
    rng = np.random.default_rng(seed)
    K_ = nmaps * per_map
    L = B.lib()
    db = C.c_void_p()
    B.check(L.sgs_kfdb_create(0, nmaps, K_, nwords + 64, C.byref(db)))
    bows = [K.random_bow(rng, nvoc, nwords - 50, nwords + 50) for _ in range(K_)]
    cap = nwords + 64
    w = np.zeros((K_, cap), np.int32); v = np.zeros((K_, cap)); n = np.zeros(K_, np.int32)
    for i, (ids, vals) in enumerate(bows):
        w[i, :len(ids)] = ids; v[i, :len(ids)] = vals; n[i] = len(ids)
    slots = np.arange(K_, dtype=np.int32); maps = (slots // per_map).astype(np.int32)
    dw, dv, dn = torch.from_numpy(w).cuda(), torch.from_numpy(v).cuda(), torch.from_numpy(n).cuda()
    B.check(L.sgs_kfdb_add(db, K_, B._p(slots), B._p(maps), dw.data_ptr(), dv.data_ptr(), dn.data_ptr(), cap, None))
    covis = np.full((K_, 10), -1, np.int32)
    for s in range(K_):
        base = (s // per_map) * per_map
        covis[s] = base + (s - base + np.arange(1, 11)) % per_map       # ten neighbours in the same map
    # each row: a key frame of its map with a third of its words replaced (a frame near that key frame)
    F = nmaps
    qw = np.zeros((F, cap), np.int32); qv = np.zeros((F, cap)); qn = np.zeros(F, np.int32); qb = []
    for f in range(F):
        ids, _ = bows[f * per_map + int(rng.integers(per_map))]
        keep = ids[rng.uniform(size=len(ids)) > 0.33]
        new = np.setdiff1d(rng.choice(nvoc, len(ids) - len(keep), replace=False), keep)
        ids2, vals2 = K.normalized(np.concatenate([keep, new]), rng.uniform(0.05, 1.0, len(keep) + len(new)))
        qw[f, :len(ids2)] = ids2; qv[f, :len(ids2)] = vals2; qn[f] = len(ids2); qb.append((ids2, vals2))
    dqw, dqv, dqn = torch.from_numpy(qw).cuda(), torch.from_numpy(qv).cuda(), torch.from_numpy(qn).cuda()
    dcov = torch.from_numpy(covis).cuda()
    cc = 64
    cand = torch.zeros((F, cc), dtype=torch.int32, device='cuda'); nc = torch.zeros(F, dtype=torch.int32, device='cuda')
    st = torch.zeros((F, 4), dtype=torch.int32, device='cuda')
    qm = np.arange(F, dtype=np.int32)
    s = torch.cuda.current_stream().cuda_stream

    def call():
        B.check(L.sgs_kfdb_reloc_candidates_device(db, F, B._p(qm), dqw.data_ptr(), dqv.data_ptr(), dqn.data_ptr(), cap, dcov.data_ptr(), cand.data_ptr(), cc,
                                                   nc.data_ptr(), st.data_ptr(), C.c_void_p(s)))
    for _ in range(20):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        call()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    # the restatement on the CPU, the same queries (rows up to cpu_rows), checked against the device's last call
    ref = K.Database(K_)
    for i in range(K_):
        ref.add(i, int(maps[i]), *bows[i])
    ncpu = min(F, cpu_rows)
    t0 = time.perf_counter()
    want = [ref.query(f, *qb[f], covis, cc) for f in range(ncpu)]
    cpu_ms = (time.perf_counter() - t0) * 1e3 * F / ncpu
    got_c, got_n, got_s = cand.cpu().numpy(), nc.cpu().numpy(), st.cpu().numpy()
    same = all(list(got_s[f]) == want[f][1] and list(got_c[f, :got_n[f]]) == want[f][0][:cc] for f in range(ncpu))
    L.sgs_kfdb_destroy(db)
    return dict(rows=F, keyframes_per_map=per_map, words=nwords, device_ms_per_call=round(ms, 4), restatement_cpu_ms_per_call=round(cpu_ms, 1),
                cpu_rows_timed=ncpu, equal_to_restatement=bool(same), mean_sharing=float(got_s[:, 0].mean()), mean_scored=float(got_s[:, 2].mean()))


if __name__ == '__main__':
    import ctypes as C
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--cpu-rows', type=int, default=8)
    a = ap.parse_args()
    name, power = card()
    res = [case(64, 1024, 20000, 700, a.iters, a.cpu_rows, 1), case(1, 8192, 20000, 700, a.iters, 1, 2)]
    print(json.dumps(dict(card=name, power_limit=power, cases=res)))
