"""The named PoseOptimization inputs shared by the tests of the CPU restatement (oracle/pose_opt.cpp) and of the device kernel (pose_opt.cu).

Each case is (family, name, scenario) with the scenario in the `scenarios.pose_scenario` dict format.  `reference_cases()` are the frames the
restatement is pinned on against the reference's own Optimizer.cc + g2o; `designed_cases()` add inputs chosen so that plausible one-line slips in
the Levenberg schedule, the Huber rounds or the round structure change the result (tests/test_pose_opt_cases.py checks that they do).  A single
inv_level_sigma2 table serves every case: the 8-level cases read its first eight entries, which equal the 8-level table."""
import numpy as np

import scenarios as S

NLEVELS = 16
_SF = S.scale_factors(NLEVELS)
INV_S2 = (1.0 / (_SF * _SF)).astype(np.float32)             # 1 / sigma^2 of a 16-level 1.2 pyramid, as pose_scenario computes it; INV_S2[:8] is the 8-level table


def _sub(s, k):
    """The scenario with only its first k keypoints holding a map point."""
    s = dict(s); s['has'] = np.zeros_like(s['has']); s['has'][:k] = 1
    return s


def reference_cases():
    """The 61 frames of tests/test_optimizer_ref.py."""
    out = [('plain', 'plain%d' % seed, S.pose_scenario(seed)) for seed in range(1, 25)]
    out += [('hard', 'hard%d' % seed, S.pose_scenario(seed, outlier_frac=0.45, noise=1.5, pose_err=(0.08, 0.3))) for seed in range(30, 42)]
    # a start far from the optimum: Levenberg rejects trials and raises lambda
    out += [('far', 'far%d' % seed, S.pose_scenario(seed, n=300, outlier_frac=0.3, noise=1.0, pose_err=(0.25, 0.8))) for seed in range(42, 48)]
    for seed in (50, 51, 52):
        out += [('mono', 'mono%d' % seed, S.pose_scenario(seed, mono_frac=1.0)), ('stereo', 'stereo%d' % seed, S.pose_scenario(seed, mono_frac=0.0))]
    base = S.pose_scenario(5, outlier_frac=0.0, noise=0.2)
    out += [('few', 'few%d' % k, _sub(base, k)) for k in (0, 1, 2)]                     # < 3 correspondences: pose untouched, 0 returned
    out += [('edges', 'edges%d' % k, _sub(base, k)) for k in (3, 4, 6, 9, 10, 11, 14)]  # < 10 edges: a single round; 10 and more: four
    tiny = S.pose_scenario(7, n=12, outlier_frac=0.5, noise=2.0); tiny['has'][:] = 1     # a tiny graph with outliers
    out.append(('tiny', 'tiny7', tiny))
    behind = S.pose_scenario(9); behind['xyz'][:40] *= -1                                # negative depth: huge residuals, flagged in the first round
    out.append(('behind', 'behind9', behind))
    out.append(('exact', 'exact11', S.pose_scenario(11, outlier_frac=0.0, noise=0.0, pose_err=(0.0, 0.0))))   # already at the optimum
    return out


def _small(seed, k):
    s = S.pose_scenario(seed, n=k, outlier_frac=0.3, noise=1.5); s['has'][:] = 1
    return s


# Seeds picked from a scan of the family's parameters (seeds 100-199) for the property named, which tests/test_pose_opt_cases.py keeps checked:
# an iteration rejects more than five Levenberg trials in a row (REJECT_SEEDS: a far start), and g2o's "three bad iterations" exit fires with the
# 1e3 factor and would not with 1e4 (NBAD_SEEDS: 16 edges, 30 % outliers, 1.5 px noise).
REJECT_SEEDS = (101, 104)
NBAD_SEEDS = (174, 179)


def designed_cases():
    out = []
    # far starts, 30 % outliers: several rejected trials per iteration, outlier sets that move from round to round
    for i, n in enumerate((200, 500, 900)):
        for j, rot in enumerate((0.2, 0.25, 0.3, 0.3)):
            seed = 200 + 4 * i + j
            out.append(('farstart', 'farstart%d_%d' % (n, seed), S.pose_scenario(seed, n=n, outlier_frac=0.3, noise=1.0, pose_err=(rot, 0.6))))
    # exactly 9 edges (one round) and exactly 10 (four rounds), with outliers
    for seed in range(300, 306):
        out.append(('nine', 'nine%d' % seed, _small(seed, 9)))
        out.append(('ten', 'ten%d' % seed, _small(seed, 10)))
    # a 16-level pyramid: octaves 8-15 read the upper half of the sigma table
    for seed in (400, 401, 402):
        out.append(('levels16', 'levels16_%d' % seed, S.pose_scenario(seed, n=600, outlier_frac=0.2, noise=0.8, nlevels=NLEVELS)))
    for seed in REJECT_SEEDS:
        out.append(('rejects', 'rejects%d' % seed, S.pose_scenario(seed, n=300, outlier_frac=0.3, noise=1.0, pose_err=(0.3, 0.6))))
    for seed in NBAD_SEEDS:
        out.append(('nbad', 'nbad%d' % seed, _small(seed, 16)))
    out.append(('stale', 'stale207', stale_error_case()))
    return out


def stale_error_case():
    """farstart500_207 with one monocular octave-0 edge added whose first round ends on ten rejected Levenberg trials.  The edge's chi2 at the
    last TRIED estimate (what g2o's classification reads) is 5.99100039066, at the final estimate 5.99100051605; the float compare with 5.991f
    switches at 5.99100041388, so the edge is an inlier after the first round by the stale error and would be an outlier by a fresh one -- margins
    of 2.3e-8 and 1.0e-7, far above the ~1e-12 the device and the restatement differ by.  The stale chi2 rounds to exactly 5.991f, so the edge
    also decides between `chi2 > 5.991f` and `>=`.  Found by a search over the edge's position and a secant on its observation; the point and
    the observation are stored as float32."""
    s = S.pose_scenario(207, n=500, outlier_frac=0.3, noise=1.0, pose_err=(0.3, 0.6))
    s['xyz'] = np.vstack([s['xyz'], np.array([[-0.03472725674510002, 1.0659193992614746, 2.770528554916382]], np.float32)])
    s['xy'] = np.vstack([s['xy'], np.array([[322.4154968261719, 415.0]], np.float32)])
    s['octave'] = np.r_[s['octave'], 0].astype(np.int32); s['uright'] = np.r_[s['uright'], -1].astype(np.float32); s['has'] = np.r_[s['has'], 1].astype(np.uint8)
    return s


def all_cases():
    return reference_cases() + designed_cases()


def ulp_distance(a, b):
    """Element-wise distance of two float32 arrays in units in the last place: the number of float32 values between them (0 = identical bits,
    +0 and -0 count as equal)."""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    return np.abs(ordered(a) - ordered(b))
