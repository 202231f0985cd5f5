"""The greedy sampler's rule (misc/model.py:590-615) in float64, and the logit rows on which an implementation of it goes wrong.

The three CUDA samplers (greedy_pick_kernel, reduce_pick_kernel, MODE_PICK of wg_gemm_kernel) and their CPU transliterations in
test_sampler_emulation.py are all compared with `pick_reference` on the rows `special_rows` builds."""
import numpy as np

STEP = 0.125          # every logit is a multiple of 1/8 in [-12, 12]: exact in fp32, tf32 and fp16, and so is any split of it


def pick_reference(logits, unk):
    """logits [B, V] float64 -> (token [B] int64, logp [B] float64): top-2 with the lower index winning ties, the runner-up when the
    winner is `unk`, log-softmax value of the token taken."""
    logits = np.asarray(logits, np.float64)
    B, V = logits.shape
    top2 = np.argsort(-logits, axis=1, kind="stable")[:, :2]          # stable: equal values keep ascending index order
    rows = np.arange(B)
    take = np.where(top2[:, 0] != unk, top2[:, 0], top2[:, 1])
    m = logits.max(axis=1)
    lse = m + np.log(np.exp(logits - m[:, None]).sum(axis=1))
    return take.astype(np.int64), logits[rows, take] - lse


def top2_gap(logits, unk):
    """Distance between the value of the token `pick_reference` takes and the best other candidate it could have taken."""
    logits = np.asarray(logits, np.float64)
    s = -np.sort(-logits, axis=1)
    top = np.argmax(logits, axis=1)
    return np.where(top != unk, s[:, 0] - s[:, 1], s[:, 1] - s[:, 2] if logits.shape[1] > 2 else np.inf)


KINDS = ("unique_max", "unk_max", "tie_in_tile", "tie_across_tiles", "tie_across_1024", "tie_across_warps", "tie_unk_lower", "tie_unk_higher",
         "three_way_tie", "unk_max_tie_second", "all_equal", "max_last_column", "max_last_tile", "unk_runner_up", "random")


def special_rows(B, V, unk, seed):
    """[B, V] float64 logits, row b of kind KINDS[b % len(KINDS)].  The background is random multiples of 1/8 in [-12, 8] (so it has
    plenty of ties of its own below the top); the row's kind places the values 10 / 9 on top of it.  A kind that does not fit V (a pair
    1024 columns apart in a 301-word vocabulary) leaves the random row."""
    rs = np.random.RandomState(seed)
    x = rs.randint(-96, 65, size=(B, V)).astype(np.float64) * STEP
    kinds = []

    def cols(n, lo=0, hi=V):
        """n distinct ascending columns in [lo, hi) that are not unk, or None"""
        pool = [c for c in range(lo, min(hi, V)) if c != unk]
        if len(pool) < n:
            return None
        return sorted(rs.choice(pool, size=n, replace=False).tolist())

    def pair(dist):
        pool = [c for c in range(V - dist) if c != unk and c + dist != unk]
        if not pool:
            return None
        c = int(rs.choice(pool))
        return c, c + dist

    for b in range(B):
        kind = KINDS[b % len(KINDS)]
        kinds.append(kind)
        r = x[b]
        if kind == "unique_max":
            c = cols(1)
            if c: r[c[0]] = 10
        elif kind == "unk_max":
            c = cols(1)
            r[unk] = 10
            if c: r[c[0]] = 9
        elif kind == "tie_in_tile":
            t0 = 64 * int(rs.randint(0, (V + 63) // 64))
            c = cols(2, t0, t0 + 64)
            if c: r[c] = 10
        elif kind in ("tie_across_tiles", "tie_across_1024", "tie_across_warps"):
            c = pair({"tie_across_tiles": 64, "tie_across_1024": 1024, "tie_across_warps": 32}[kind])
            if c: r[list(c)] = 10
        elif kind == "tie_unk_lower":
            c = cols(1, 0, unk)
            if c: r[[c[0], unk]] = 10
        elif kind == "tie_unk_higher":
            c = cols(1, unk + 1, V)
            if c: r[[unk, c[0]]] = 10
        elif kind == "three_way_tie":
            c = cols(3)
            if c: r[c] = 10
        elif kind == "unk_max_tie_second":
            c = cols(2)
            if c:
                r[unk] = 10
                r[c] = 9
        elif kind == "all_equal":
            r[:] = float(rs.randint(-96, 97)) * STEP
        elif kind == "max_last_column":
            r[V - 1] = 10
        elif kind == "max_last_tile":
            c = cols(1, (V - 1) // 64 * 64, V)
            if c: r[c[0]] = 10
        elif kind == "unk_runner_up":
            c = cols(1)
            if c:
                r[c[0]] = 10
                r[unk] = 9
    return x, kinds
