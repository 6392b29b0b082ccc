"""The batched carries of the scatters' tile adds (transfer_kernels.cu, tile_add_lo): on the fast path a head issues the low-word adds of
several faces back to back and only then the high-word adds, each the high half of its value plus the carry out of its own low-word add,
and it adds zeros rather than branch around them.  Between a lane's low add and its high add any number of other adds (other lanes, other
warps, other batches) reach the same words.  Whatever the interleaving, (hi << 32) | lo must be the int64 sum modulo 2^64, bit for bit."""
import numpy as np

M32 = 0xFFFFFFFF


def batched_tile_sums(streams, nwords, rng):
    """Emulates the tile words under concurrent batched adds.  streams: per adder a list of batches, a batch a list of (word, q).  An adder
    runs a batch as: every low-word add (32-bit atomic add returning the old word) in order, then every high-word add of that batch; the
    adders' single atomic operations interleave in the order rng picks."""
    lo, hi = [0] * nwords, [0] * nwords

    def ops(batches):
        for batch in batches:
            carry = []
            for w, q in batch:
                ql = q & M32
                old = lo[w]
                lo[w] = (old + ql) & M32
                carry.append((w, (((q >> 32) & M32) + (1 if old + ql > M32 else 0)) & M32))
                yield
            for w, h in carry:
                hi[w] = (hi[w] + h) & M32
                yield

    live = [ops(s) for s in streams]
    while live:
        k = int(rng.integers(len(live)))
        try:
            next(live[k])
        except StopIteration:
            live.pop(k)
    out = []
    for w in range(nwords):
        s = (hi[w] << 32) | lo[w]
        out.append(s - (1 << 64) if s >> 63 else s)
    return out


def int64_sums(streams, nwords):
    acc = [0] * nwords
    for s in streams:
        for batch in s:
            for w, q in batch:
                acc[w] += q
    return [((a + (1 << 63)) % (1 << 64)) - (1 << 63) for a in acc]


def _streams(rng, values, nwords, adders, batch):
    """Cut `values` into `adders` streams of batches of `batch` faces, each value to a random word."""
    words = rng.integers(0, nwords, len(values))
    items = [(int(w), int(q)) for w, q in zip(words, values)]
    per = [items[k::adders] for k in range(adders)]
    return [[s[i:i + batch] for i in range(0, len(s), batch)] for s in per]


def test_batched_carries_equal_the_int64_sums_on_adversarial_values():
    rng = np.random.default_rng(2024)
    two63 = 1 << 63
    for trial in range(120):
        n = int(rng.integers(8, 300))
        kind = trial % 6
        if kind == 0:  # low words just below 2^32: almost every low add wraps
            v = [int(x) for x in (rng.integers(0, 1 << 20, n) << 32) | rng.integers(0xFFFFFF00, 0xFFFFFFFF, n, endpoint=True)]
        elif kind == 1:  # negative values (two's complement: high words 0xFFFFFFFF)
            v = [int(x) for x in rng.integers(-(1 << 45), 0, n)]
        elif kind == 2:  # near +-2^63: the sums wrap modulo 2^64
            v = [int(x) for x in rng.choice([two63 - 1, -two63, two63 - 2, -two63 + 1], n)]
        elif kind == 3:  # mixed signs around 0
            v = [int(x) for x in rng.integers(-(1 << 33), 1 << 33, n)]
        elif kind == 4:  # zeros among them (weights that round to 0, values left out)
            v = [int(x) if rng.random() < 0.6 else 0 for x in rng.integers(-(1 << 40), 1 << 40, n)]
        else:  # the full int64 range
            v = [int(x) for x in rng.integers(-two63, two63 - 1, n, dtype=np.int64, endpoint=True)]
        nwords = int(rng.integers(1, 9))
        streams = _streams(rng, v, nwords, adders=int(rng.integers(1, 9)), batch=int(rng.choice([1, 4, 8, 16])))
        assert batched_tile_sums(streams, nwords, rng) == int64_sums(streams, nwords), trial


def test_batched_carries_2048_adds_into_one_word():
    """2048 adds into one word from 64 adders in batches of 8: values whose low words wrap on every add, and values near -2^63, whose sum
    wraps many times over."""
    rng = np.random.default_rng(7)
    for base in (0xFFFFFFFF, -(1 << 63) + 12345):
        v = [base + int(x) for x in rng.integers(0, 1 << 12, 2048)]
        if base > 0:
            v = [x | 0xFFFFFF00 for x in v]
        streams = _streams(rng, v, 1, adders=64, batch=8)
        got = batched_tile_sums(streams, 1, rng)
        want = sum(v)
        assert got == int64_sums(streams, 1) == [((want + (1 << 63)) % (1 << 64)) - (1 << 63)]
