"""Poisons, where they go, and the comparator of the isolation tests (TEST INFRASTRUCTURE, shared by tests/test_gpu_isolation.py and
tests/test_isolation_cases_cpu.py).

Many tenants share one launch: the utterances of a padded or ragged batch, the streams of a pool, the generators of a multi-generator
pool and the voices of a VoiceBank.  A kernel that reads a neighbour's data and then cancels it with a zero (a mask, a discarded
accumulator, P = 0, a zero tap) gives the same bits on finite data, since 0 * x = 0, but 0 * NaN = NaN and 0 * Inf = NaN.  So the
isolation tests put non-finite and extreme values into one tenant and ask that every other tenant's output is the same as in the clean
run, and that the poisoned tenant's output is the same as its own solo call with the same poison.  `same` is that equality: NaN where
NaN, the same infinities, and every finite element bit for bit (an int32 view, so -0 and +0 differ)."""
import torch

NAN, INF = float("nan"), float("inf")
# NaN and both infinities; 65504, the fp16 maximum, where the tensor-core operand split saturates; 3e38, where fp32 sums overflow
POISONS = {"nan": NAN, "+inf": INF, "-inf": -INF, "f16max": 65504.0, "f32big": 3e38}
TILE = 128                                             # rows per tile of the tensor-core conv and the fused kernels' output tiles
PLACEMENTS = ("first", "last", "boundary", "frame", "channel")


def same(a, b):
    """True when a and b have the same shape and dtype, NaN in the same places, the same infinities, and every other element bit for
    bit equal.  Integer tensors compare as integers."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if not a.dtype.is_floating_point:
        return bool(torch.equal(a, b))
    a32, b32 = a.float(), b.float()
    na, nb = torch.isnan(a32), torch.isnan(b32)
    if not torch.equal(na, nb):
        return False
    fa, fb = torch.where(na, 0.0, a32).contiguous(), torch.where(nb, 0.0, b32).contiguous()
    return bool(torch.equal(fa.view(torch.int32), fb.view(torch.int32)))


def diff(a, b):
    """A one-line account of how a and b differ, for assertion messages."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return f"shape / dtype {tuple(a.shape)} {a.dtype} vs {tuple(b.shape)} {b.dtype}"
    if not a.dtype.is_floating_point:
        return f"{int((a != b).sum())} elements differ"
    a, b = a.float(), b.float()
    na, nb = torch.isnan(a), torch.isnan(b)
    fin = torch.isfinite(a) & torch.isfinite(b)
    err = (a - b)[fin].abs().max().item() if bool(fin.any()) else 0.0
    return (f"NaN {int(na.sum())} vs {int(nb.sum())} ({int((na != nb).sum())} differ), inf {int(torch.isinf(a).sum())} vs "
            f"{int(torch.isinf(b).sum())}, finite max |diff| {err:.3g}")


def rows(n, boundary):
    """The rows to poison in an utterance of n live rows: {placement: row}.  'first' and 'last' are rows 0 and n - 1; 'boundary' is the
    given row on a tile (and chunk) boundary, when it is live; 'frame' and 'channel' are the boundary row (else the middle row),
    'frame' to be poisoned across all channels and 'channel' in one channel only."""
    mid = boundary if 0 < boundary < n else n // 2
    out = {"first": 0, "last": n - 1, "frame": mid, "channel": mid}
    if 0 < boundary < n:
        out["boundary"] = boundary
    return out


def positions(B):
    """The batch positions of the poisoned tenant: first, middle and last, so that both of its neighbours are exercised."""
    return sorted({0, B // 2, B - 1})


def cases(B, n_of, boundary, poisons=tuple(POISONS)):
    """(poison name, batch position, placement, row) tuples: every poison at every position, and the placements cycling through them,
    so that with all five poisons every (position, placement) pair runs once.  n_of(b) is tenant b's live row count."""
    out, i = [], 0
    for p in poisons:
        for q in positions(B):
            rs = rows(n_of(q), boundary)
            names = [k for k in PLACEMENTS if k in rs]
            k = names[i % len(names)]
            out.append((p, q, k, rs[k]))
            i += 1
    return out


def poison(x, b, row, value, placement, axis=1, channel=0):
    """A copy of x with tenant b's `row` along `axis` (1: [B, T, C] channels-last, 2: [B, C, T]) set to value: every channel for a
    row placement, channel `channel` only for 'channel'."""
    x = x.clone()
    idx = [b, slice(None), slice(None)][:x.dim()]
    idx[axis] = row
    if placement == "channel" and x.dim() == 3:
        idx[3 - axis] = min(channel, x.shape[3 - axis] - 1)
    x[tuple(idx)] = value
    return x
