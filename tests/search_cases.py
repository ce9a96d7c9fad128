"""lk_search_poses restated on the host: the candidate lattice of include/legkilo_b200.h in numpy, and the composition the
call equals (lk_score_poses wide, the best k per set, lk_refine_poses, lk_score_poses tight, the order by tight count).

Shared by tests/test_gpu_search_poses.py, tests/test_search_poses_cpu.py and tools/search_poses_timing.py."""
import numpy as np

from legkilo_b200 import abi, synth

# wide blocks of the recipe's search, tight blocks of its final check (INTEGRATION.md §5)
WIDE_ROT, WIDE_POS = (np.deg2rad(2.0) ** 2) * np.eye(3), 0.1 ** 2 * np.eye(3)
TIGHT_ROT, TIGHT_POS = (np.deg2rad(0.2) ** 2) * np.eye(3), 0.01 ** 2 * np.eye(3)


def lattice_at(att, origin, step, counts, c):
    """Candidates c (int array) of one set: att [n_att, 3, 3] (or [n_att, 9]), origin [3], step [3], counts (nx, ny, nz).
    Returns rot [n, 3, 3], pos [n, 3]: candidate c is attitude c // L at lattice point (ix, iy, iz) of r = c % L, ix
    fastest, pos = origin + i * step (numpy rounds the product, then the sum)."""
    att = np.asarray(att, np.float64).reshape(-1, 3, 3)
    nx, ny, nz = (int(v) for v in counts)
    L = nx * ny * nz
    c = np.asarray(c, np.int64)
    a, r = c // L, c % L
    i = np.stack([r % nx, (r // nx) % ny, r // (nx * ny)], 1).astype(np.float64)
    return att[a], np.asarray(origin, np.float64)[None, :] + i * np.asarray(step, np.float64)[None, :]


def lattice(att, origin, step, counts, first=0, n=None):
    """Candidates [first, first + n) of one set (all of them by default), as lattice_at."""
    n = len(np.asarray(att).reshape(-1, 9)) * int(np.prod(np.asarray(counts, np.int64))) - first if n is None else n
    return lattice_at(att, origin, step, counts, np.arange(first, first + n, dtype=np.int64))


def yaw_attitudes(yaws_deg, R0=np.eye(3)):
    return np.array([synth.exp_so3((0.0, 0.0, np.deg2rad(y))) @ R0 for y in yaws_deg])


def keys(counts, first):
    """The total order of the keep: count descending, candidate index ascending, as one ascending uint64 key."""
    cnt = np.asarray(counts).astype(np.uint64)
    return ((np.uint64(0xFFFFFFFF) - cnt) << np.uint64(32)) | (np.arange(len(cnt), dtype=np.uint64) + np.uint64(first))


def compose(eng, pts, set_offsets, att_offsets, att, origin, step, counts, iters, k, rot_cov=WIDE_ROT, pos_cov=WIDE_POS,
            rot_cov_tight=TIGHT_ROT, pos_cov_tight=TIGHT_POS, slice_=None):
    """The composition lk_search_poses equals, through the public calls. slice_: score each set's candidates in slices of
    that many, merging the best k on the host. Returns what search_poses returns."""
    so, ao = np.asarray(set_offsets, np.int64), np.asarray(att_offsets, np.int64)
    att = np.asarray(att, np.float64).reshape(-1, 3, 3)
    n_sets = len(so) - 1
    L = int(np.prod(np.asarray(counts, np.int64)))
    kept_rot, kept_pos, kept_c = [], [], []
    if slice_ is None:  # steps 1-2 as the recipe runs them: every candidate of every set in one lk_score_poses call
        cands = [lattice(att[ao[s]:ao[s + 1]], origin[s], step, counts) for s in range(n_sets)]
        n = [len(r) for r, _ in cands]
        rec = eng.score_poses(pts, so.astype(np.uint32), np.repeat(np.arange(n_sets), n).astype(np.uint32),
                              np.concatenate([r for r, _ in cands]), np.concatenate([p for _, p in cands]), rot_cov, pos_cov)
        first = np.concatenate([[0], np.cumsum(n)])
        for s in range(n_sets):
            c = np.argsort(-rec[first[s]:first[s + 1], abi.SCORE_COUNT], kind="stable")[:k]
            kept_rot.append(cands[s][0][c])
            kept_pos.append(cands[s][1][c])
            kept_c.append(c)
    for s in range(n_sets if slice_ is not None else 0):  # steps 1-2 in slices, the best k merged on the host
        A = att[ao[s]:ao[s + 1]]
        N, sl = len(A) * L, slice_
        best = np.zeros(0, np.uint64)
        for f in range(0, N, sl):
            rot, pos = lattice(A, origin[s], step, counts, f, min(sl, N - f))
            rec = eng.score_poses(pts[so[s]:so[s + 1]], [0, so[s + 1] - so[s]], np.zeros(len(rot), np.uint32), rot, pos,
                                  rot_cov, pos_cov)
            best = np.sort(np.concatenate([best, keys(rec[:, abi.SCORE_COUNT], f)]))[:k]
        c = (best & np.uint64(0xFFFFFFFF)).astype(np.int64)
        rot, pos = lattice_at(A, origin[s], step, counts, c)
        kept_rot.append(rot)
        kept_pos.append(pos)
        kept_c.append(c)
    rot, pos = np.concatenate(kept_rot), np.concatenate(kept_pos)
    ps = np.repeat(np.arange(n_sets), k).astype(np.uint32)
    ro, po, _ = eng.refine_poses(pts, so.astype(np.uint32), ps, rot, pos, rot_cov, pos_cov, iters, want_records=False)
    rec = eng.score_poses(pts, so.astype(np.uint32), ps, ro, po, rot_cov_tight, pos_cov_tight)
    out = [np.zeros((n_sets, k, 3, 3)), np.zeros((n_sets, k, 3)), np.zeros((n_sets, k, abi.SCORE_STRIDE)),
           np.zeros((n_sets, k), np.uint32)]
    for s in range(n_sets):
        g = np.arange(s * k, (s + 1) * k)
        o = g[np.argsort(-rec[g, abi.SCORE_COUNT], kind="stable")]
        out[0][s], out[1][s], out[2][s], out[3][s] = ro[o], po[o], rec[o], np.asarray(kept_c[s])[o - s * k]
    return tuple(out)


def same(a, b):
    """Bitwise equality of two search results."""
    return all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(a, b))
