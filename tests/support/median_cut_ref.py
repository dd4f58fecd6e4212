"""Restatement of compression.median_cut, box by box, with the orders numpy leaves implicit spelled out:

  * within a box the points are ordered by (key on the split axis, original index): a stable sort of the box in index
    order, where numpy's float order makes -0.0 == +0.0 and puts NaN last;
  * np.add.reduceat of a segment is its first element plus numpy's pairwise sum of the rest (blocks of < 8 summed in
    order from -0.0, blocks of <= 128 with eight accumulators, longer runs split at a multiple of 8 below the half);
  * np.cumsum over the sorted array is one sequential fp64 sum running through every box in box order;
  * np.bincount sums in index order.

Each order has a perturbed variant, so tests can show a fixture tells the true order from a wrong one:
tie="reverse" (ties by descending index), total="sequential", cum="pairwise" (each box's running sum restarted and
summed pairwise), axis="last" (last argmax).
"""
import numpy as np


def pairwise_sum(a):
    n = len(a)
    if n < 8:
        r = -0.0
        for v in a:
            r += float(v)
        return r
    if n <= 128:
        r = [float(v) for v in a[:8]]
        i = 8
        while i < n - n % 8:
            for k in range(8):
                r[k] += float(a[i + k])
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for v in a[i:]:
            res += float(v)
        return res
    h = n // 2
    h -= h % 8
    return pairwise_sum(a[:h]) + pairwise_sum(a[h:])


def sequential_sum(a):
    r = 0.0
    for v in a:
        r += float(v)
    return r


def reduceat_sum(a):
    """np.add.reduceat(a, [0])[0] for a non-empty segment"""
    return float(a[0]) if len(a) == 1 else float(a[0]) + pairwise_sum(a[1:])


def _axis(ext, axis):
    if axis == "first":
        return int(np.argmax(ext))
    return 2 - int(np.argmax(ext[::-1]))


def median_cut_ref(points, bits, weights=None, tie="index", total="reduceat", cum="sequential", axis="first"):
    pts = np.ascontiguousarray(points, dtype=np.float32)
    n = pts.shape[0]
    n_colors = 1 << bits
    if n == 0:
        return np.zeros((n_colors, 3), np.float32), np.zeros((0,), np.int64)
    w = None if weights is None or len(weights) == 0 else np.asarray(weights, dtype=np.float64)
    box = np.zeros(n, dtype=np.int64)
    for _ in range(bits):
        new_box = 2 * box
        running = 0.0
        for bid in np.unique(box):
            members = np.flatnonzero(box == bid)                      # index order
            P = pts[members]
            ext = P.max(axis=0) - P.min(axis=0)                       # NaN propagates like maximum.reduceat
            ax = _axis(ext, axis)
            key = P[:, ax]
            if tie == "index":
                order = np.argsort(key, kind="stable")
            else:
                order = (len(key) - 1 - np.argsort(key[::-1], kind="stable"))
            m = len(members)
            splittable = ext[ax] > 0
            if w is None:
                up_sorted = np.arange(m) >= (m + 1) // 2
            else:
                ws = w[members[order]]
                tot = reduceat_sum(ws) if total == "reduceat" else sequential_sum(ws)
                base = running
                up_sorted = np.zeros(m, bool)
                for j in range(m):
                    if cum == "sequential":
                        running += float(ws[j])
                        c = running - base
                    else:
                        c = pairwise_sum(ws[:j + 1])
                    up_sorted[j] = j > 0 and c > 0.5 * tot
                if cum != "sequential":
                    running += sequential_sum(ws)
            if splittable:
                new_box[members[order]] += up_sorted
        box = new_box
    palette = np.zeros((n_colors, 3), dtype=np.float64)
    cnt = np.zeros(n_colors, dtype=np.float64)
    for i in range(n):                                                # np.bincount: index order
        wi = 1.0 if w is None else float(w[i])
        cnt[box[i]] += wi
        for c in range(3):
            palette[box[i], c] += float(pts[i, c]) if w is None else float(pts[i, c]) * wi
    palette /= np.maximum(cnt, 1e-30)[:, None]
    palette[cnt == 0] = 0.0
    return palette.astype(np.float32), box


def same(a, b):
    """palettes and maps equal bit for bit (NaN palette entries compare by their bits)"""
    return np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


def fixtures():
    """name -> (points [n, 3] f32, bits, weights or None): small point sets on which the host's result differs from
    every perturbed variant that applies (tie and axis rules; for weighted sets also the total and the running sum)"""
    rs = np.random.RandomState(7)
    f = {}
    # fp16-valued coordinates with many duplicates on every axis: ties decide the split
    q = (rs.randint(-6, 7, size=(600, 3)) / 4).astype(np.float16).astype(np.float32)
    f["dup_fp16"] = (q, 6, None)
    # equal extents on two axes, so the axis rule decides
    e = rs.randint(0, 5, size=(400, 3)).astype(np.float32)
    e[:, 1] = rs.randint(0, 3, size=400)
    f["equal_extents"] = (e, 5, None)
    # signed zeros and infinities among duplicates
    z = (rs.randint(-2, 3, size=(300, 3)) * 0.5).astype(np.float32)
    z[rs.rand(300, 3) < 0.2] = -0.0
    z[5, 0], z[9, 1], z[17, 2] = np.inf, -np.inf, np.inf
    f["signed_zeros_inf"] = (z, 6, None)
    # weights of mixed magnitudes one ulp apart: the order of the fp64 sums decides the threshold
    ra = np.random.RandomState(2)
    a = (ra.randint(-6, 7, size=(300, 3)) / 4).astype(np.float32)
    wa = ra.choice([1.0, 3.0, 2.0 ** -30, 0.1, 1e8], size=300) * ra.choice([1, 1 + 2 ** -52], size=300)
    f["weights_adversarial"] = (a, 5, wa)
    return f
