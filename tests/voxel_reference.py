"""Pure-numpy statements of the two data-parallel reformulations the GPU voxel pipeline relies on
(ouster-sdk_b200/csrc/ob_voxel.cu), so the CPU tests can check them against the oracle's sequential loops:

  * xorshift32 (seed 42) jumped ahead with GF(2) matrices: state after k steps = M^k * 42;
  * the forward Fisher-Yates shuffle of core::voxel_downsample resolved without a serial loop.
"""
import numpy as np

MASK = 0xFFFFFFFF


def xs_step(s):
    s ^= (s << 13) & MASK
    s ^= s >> 17
    s ^= (s << 5) & MASK
    return s


def _apply(cols, v):
    """GF(2) matrix (32 columns, column j = image of 1 << j) times the vectors v."""
    r = np.zeros_like(v)
    for j in range(32):
        r ^= np.where((v >> np.uint64(j)) & np.uint64(1), cols[j], np.uint64(0))
    return r


def jump_table():
    m = np.zeros((40, 32), np.uint64)
    m[0] = [xs_step(1 << j) for j in range(32)]
    for b in range(1, 40):
        m[b] = _apply(m[b - 1], m[b - 1].copy())
    return m


_JUMP = jump_table()


def xs_state_after(steps):
    """State of xorshift32 seeded with 42 after `steps` steps (vectorised over an integer array)."""
    steps = np.asarray(steps, np.uint64)
    v = np.full(steps.shape, 42, np.uint64)
    for b in range(40):
        sel = ((steps >> np.uint64(b)) & np.uint64(1)).astype(bool)
        if sel.any():
            v = np.where(sel, _apply(_JUMP[b], v), v)
    return v


def parallel_shuffle(n):
    """Input index of the element that the reference's shuffle (voxel_hash_map.cpp:281-290) leaves at each
    position, computed from the per-step draws alone: step s swaps s and j_s; the element ending at i is
    f(pred(i)) if an earlier step chose j_i too (pred(i) = the last one), else j_i; f(p) = p unless a step
    s < p chose j_s = p, then f(L(p)) with L(p) the last such step."""
    if n == 0:
        return np.empty(0, np.int64)
    s = np.arange(n, dtype=np.uint64)
    rnd = xs_state_after(s + np.uint64(1))
    j = (s + ((rnd * (np.uint64(n) - s)) >> np.uint64(32))).astype(np.int64)
    j[n - 1] = n - 1
    order = np.argsort(j, kind="stable")           # steps grouped by j, ascending s inside a group
    sj = j[order]
    where = np.empty(n, np.int64)
    where[order] = np.arange(n)
    last_of = np.full(n, -1, np.int64)
    ends = np.r_[sj[1:] != sj[:-1], True]
    last_of[sj[ends]] = np.nonzero(ends)[0]
    out = np.empty(n, np.int64)
    for i in range(n):
        q = where[i]
        if q == 0 or sj[q - 1] != sj[q]:
            out[i] = sj[q]
            continue
        e = order[q - 1]
        while True:
            ql = last_of[e]
            if ql < 0:
                break
            st = order[ql]
            if st == e:
                if ql == 0 or sj[ql - 1] != e:
                    break
                st = order[ql - 1]
            e = st
        out[i] = e
    return out


def voxel_keys(points, voxel_size):
    """int32 voxel coordinates with x86 cvttsd2si semantics (NaN / out of range -> INT32_MIN)."""
    f = np.floor(np.asarray(points, np.float64)[:, :3] * (1.0 / voxel_size))
    ok = (f >= -2147483648.0) & (f < 2147483648.0)
    return np.where(ok, np.where(ok, f, 0).astype(np.int64), -2147483648).astype(np.int32)


def random_by_draw_index(points, voxel_size, max_pts):
    """RANDOM restated as the GPU computes it: rank in voxel -> "bucket full" flag -> exclusive scan = draw
    index k -> state M^(k+1)*42 -> slot, last writer wins.  Returns the source rows, voxels in first-appearance
    order, slots in order."""
    keys = voxel_keys(points, voxel_size)
    _, first, inv = np.unique(keys, axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    rank = np.empty(len(keys), np.int64)
    seen = {}
    for i, v in enumerate(inv):
        rank[i] = seen.get(v, 0)
        seen[v] = rank[i] + 1
    full = rank >= max_pts
    draw = np.cumsum(full) - full
    rnd = xs_state_after(draw.astype(np.uint64) + np.uint64(1))
    slot_of = np.where(full, ((rnd * np.uint64(max_pts)) >> np.uint64(32)).astype(np.int64), rank)
    buckets = {}
    for i in range(len(keys)):
        buckets.setdefault(inv[i], {})[slot_of[i]] = i
    rows = []
    for v in np.argsort(first, kind="stable"):
        b = buckets[v]
        rows += [b[k] for k in sorted(b)]
    return np.array(rows, np.int64)
