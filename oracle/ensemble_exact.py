"""A numpy float32 restatement of pnp_native_labels_ensemble (csrc/resample.cu, include/pnp_b200.h "native-grid labels of an
ensemble") in the kernel's operation order, built from oracle/native_exact.py's pieces, plus the seeded operands of its tests.
Test-only.

For every native voxel and every member k in ascending order: u^k = native_exact.coords of member k's map; the member covers the
voxel where native_exact.inside holds; its class scores are native_exact.class_scores; the first covering member's scores are
taken as they are and each later one's are added, one float32 addition per member and class; the label is
native_exact.first_max of the sums, and 0 where no member covers the voxel.  Each mutation flag restates one plausible kernel
bug (reverse, divide, first_cover, fma): tests/test_native_ensemble_cpu.py checks that each one changes some output."""
import numpy as np

from oracle import native_exact as N

F32 = np.float32


def ensemble_ref(scores, maps, shape, reverse=False, divide=False, first_cover=False, fma=False):
    """-> uint8 [m0, m1, m2]: native-grid labels of K members' prepared-grid class scores (fp32 [K, n0, n1, n2, C]) through their
    maps (fp32 [K, 12]).
    reverse:     the members summed in descending k;
    divide:      the sums divided by the number of covering members before the argmax;
    first_cover: every member's coverage decided by member 0's coordinate alone;
    fma:         FMA-contracted coordinates (native_exact.coords(fma=True))."""
    scores = np.asarray(scores, F32)
    maps = np.asarray(maps, F32).reshape(-1, 12)
    K, n, C = scores.shape[0], scores.shape[1:4], scores.shape[4]
    if maps.shape[0] != K:
        raise ValueError("%d score volumes but %d maps" % (K, maps.shape[0]))
    shape = tuple(int(s) for s in shape)
    total = np.zeros((C,) + shape, F32)
    count = np.zeros(shape, np.int64)
    cover0 = N.inside(N.coords(maps[0], shape, fma), n)
    for k in (range(K - 1, -1, -1) if reverse else range(K)):
        u = N.coords(maps[k], shape, fma)
        ok = cover0 if first_cover else N.inside(u, n)
        if not ok.any():
            continue
        v = N.class_scores(scores[k], u[:, ok])
        first = count[ok] == 0
        total[:, ok] = np.where(first[None], v, total[:, ok] + v)
        count[ok] += 1
    covered = count > 0
    out = np.zeros(shape, np.uint8)
    if covered.any():
        t = total[:, covered]
        if divide:
            t = t / count[covered].astype(F32)
        out[covered] = N.first_max(t).astype(np.uint8)
    return out


# ------------------------------------------------------------------------------------------------
# seeded operands of tests/test_native_ensemble_cpu.py and tests/test_native_ensemble_gpu.py's kernel cases
# ------------------------------------------------------------------------------------------------
def member_scores(kind, n, C, rng):
    """fp32 [n0, n1, n2, C] class scores of one member: `random` (standard normal), `ties` (constant planes and equal pairs,
    exact ties everywhere) or `near_ties` (class 1 is class 0 moved by a few ulp, so the argmax turns on the last bits)"""
    if kind == "ties":
        s = np.zeros(tuple(n) + (C,), F32)
        s[..., 0] = rng.randint(0, 3, n) * F32(0.5)
        s[..., 1] = s[..., 0]
        if C > 2:
            s[..., 2] = F32(0.5)
        if C > 4:
            s[..., 3] = rng.randint(0, 3, n) * F32(0.5)
            s[..., 4] = s[..., 3]
        s[n[0] // 2] = F32(0.25)
        return s
    s = rng.standard_normal(tuple(n) + (C,)).astype(F32)
    if kind == "near_ties":
        s[..., 1] = s[..., 0] + s[..., 0] * F32(2.0 ** -22) * rng.randint(-2, 3, n).astype(F32)
    return s


def member_map(kind, n, m, rng, k=0, K=1):
    """fp32 [12] map of member k of K from a native grid m to a score grid n:
    random   -- a general affine map, partial coverage;
    full     -- a slightly perturbed scaling that keeps every voxel inside;
    disjoint -- axis 0 cut into K bands, member k covering band k only;
    permuted -- u0 follows k, u1 follows i, u2 follows j;
    negative -- every axis reversed;
    edges    -- coordinates landing exactly on -0.5 (inside) and n - 0.5 (outside);
    nan      -- an infinite coefficient: NaN at k = 0 and infinite beyond, so the member covers nothing."""
    n, m = np.array(n, np.float64), np.array(m, np.float64)
    M = np.zeros((3, 4))
    if kind == "full":
        for a in range(3):
            M[a, a] = rng.uniform(0.9, 0.97) * (n[a] - 1) / max(m[a] - 1, 1)
            M[a, 3] = rng.uniform(0.0, 0.02)
    elif kind == "disjoint":
        band = m[0] / K
        for a in range(3):
            M[a, a] = (n[a] - 1) / max(m[a] - 1, 1)
        M[0, 0] = (n[0] - 1) / (band - 1) * 0.999
        M[0, 3] = -k * band * M[0, 0]
    elif kind == "edges":
        for a in range(3):
            M[a, a] = n[a] / (m[a] - 1)
            M[a, 3] = -0.5
        M[2, 2] = 0.5 + 0.0625 * k
    elif kind == "nan":
        M[0, 0], M[1, 1], M[2, 2] = 1.0, 1.0, np.inf
    elif kind == "permuted":
        M[0, 2], M[1, 0], M[2, 1] = n[0] / m[2], n[1] / m[0], n[2] / m[1]
        M[:, 3] = rng.uniform(-1.0, 0.5, 3)
    elif kind == "negative":
        for a in range(3):
            M[a, a] = -rng.uniform(0.8, 1.2) * n[a] / m[a]
            M[a, 3] = n[a] - 0.5 + rng.uniform(-0.5, 0.5)
    elif kind == "random":
        M[:, :3] = rng.uniform(-1.5, 1.5, (3, 3)) * (n[:, None] / m[None, :])
        M[:, 3] = rng.uniform(-1, n + 1)
    else:
        raise ValueError("unknown map kind %r" % (kind,))
    return M.astype(F32).reshape(-1)


def operands(tag, K, n, C, m, score_kind, map_kinds):
    """(scores fp32 [K, n0, n1, n2, C], maps fp32 [K, 12], gt uint8 [m0, m1, m2]) drawn from a seed of `tag`; map_kinds is one
    kind for every member or a list of K kinds; gt holds labels up to C + 1 (those >= C count as background)"""
    rng = np.random.RandomState(sum(map(ord, tag)))
    kinds = [map_kinds] * K if isinstance(map_kinds, str) else list(map_kinds)
    scores = np.stack([member_scores(score_kind, n, C, rng) for _ in range(K)])
    maps = np.stack([member_map(kinds[k], n, m, rng, k, K) for k in range(K)])
    gt = rng.randint(0, C + 2, m).astype(np.uint8)
    return scores, maps, gt
