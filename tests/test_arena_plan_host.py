"""The arena planner (CPU): arena_place, the placement behind the VAE forwards' lifetime-planned arena, through its debug
hook mgb_debug_arena_place, a pure host function of the loaded library (no handle, no device).

  * random lifetimes (seeded, thousands of buffers): no two buffers whose lifetimes overlap share a byte, every offset
    is 1024-aligned, the peak is at least the largest sum of live sizes and within PEAK_SLACK of it, and the same input
    gives the same offsets; for the library's placement and for the alternative one the tests run the network under;
  * a stack-shaped sequence (allocations under nested mark / release, as the UNet step allocates) gets exactly the
    bump allocator's offsets;
  * malformed input is refused."""
import ctypes as C

import numpy as np
import pytest

ALIGN = 1024
# the library's placement: peak over the largest live sum on the random cases below: 1.0001 to 1.107
PEAK_SLACK = 1.15


@pytest.fixture(scope="module")
def place():
    from marigold_b200 import _lib

    f = _lib.load().mgb_debug_arena_place   # builds when missing (nvcc cross-compiles without a GPU)

    def run(nbytes, t0, t1, placement=0):
        arrs = [np.ascontiguousarray(a, dtype=np.int64) for a in (nbytes, t0, t1)]
        off = np.zeros(len(arrs[0]), dtype=np.int64)
        p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))   # noqa: E731
        peak = f(len(off), p(arrs[0]), p(arrs[1]), p(arrs[2]), placement, p(off))
        return peak, off

    return run


def random_lifetimes(n, seed):
    """n buffers on a timeline of 2n events: sizes log-uniform from 1 KB to 64 MB (some unaligned), allocations in a
    random order, each freed after a random number of later events."""
    rng = np.random.default_rng(seed)
    nbytes = np.exp(rng.uniform(np.log(1 << 10), np.log(64 << 20), n)).astype(np.int64)
    nbytes[rng.random(n) < 0.5] //= ALIGN
    nbytes[nbytes == 0] = 1
    t0 = np.sort(rng.choice(2 * n, n, replace=False))
    life = np.maximum(1, rng.geometric(1.0 / rng.choice([4, 40, 400], n)))
    t1 = t0 + life
    return nbytes, t0, t1


def overlaps(nbytes, t0, t1, off, block=512):
    """Pairs of buffers whose lifetimes and byte ranges both overlap."""
    end = off + nbytes
    bad = []
    for a in range(0, len(off), block):
        sl = slice(a, a + block)
        live = (t0[sl, None] < t1[None, :]) & (t0[None, :] < t1[sl, None])
        mem = (off[sl, None] < end[None, :]) & (off[None, :] < end[sl, None])
        both = live & mem
        both[np.arange(both.shape[0]), np.arange(a, a + both.shape[0])] = False
        bad += [(a + i, j) for i, j in zip(*np.nonzero(both))]
    return bad


def max_live(nbytes, t0, t1):
    ev = sorted([(t, 1, b) for t, b in zip(t0, nbytes)] + [(t, 0, -b) for t, b in zip(t1, nbytes)])
    cur = best = 0
    for _, _, d in ev:           # at equal times the free (0) comes before the allocation (1)
        cur += d
        best = max(best, cur)
    return best


@pytest.mark.parametrize("placement", [0, 1])
@pytest.mark.parametrize("n,seed", [(2000, 1), (3000, 2), (500, 3)])
def test_random_lifetimes(place, n, seed, placement):
    nbytes, t0, t1 = random_lifetimes(n, seed)
    peak, off = place(nbytes, t0, t1, placement)
    assert peak == int((off + nbytes).max())
    assert (off % ALIGN == 0).all() and (off >= 0).all()
    assert not overlaps(nbytes, t0, t1, off)
    lo = max_live(nbytes, t0, t1)
    assert peak >= lo
    if placement == 0:
        assert peak <= PEAK_SLACK * lo, peak / lo
    peak2, off2 = place(nbytes, t0, t1, placement)
    assert peak2 == peak and np.array_equal(off2, off)


def test_alternative_placement_moves_buffers(place):
    nbytes, t0, t1 = random_lifetimes(1000, 4)
    _, a = place(nbytes, t0, t1, 0)
    _, b = place(nbytes, t0, t1, 1)
    assert (a != b).mean() > 0.5


def stack_sequence(seed, n_ops=4000):
    """A random stack-shaped sequence, run through a restatement of the bump allocator (net.cu Arena without a plan):
    allocations, nested marks and releases to the innermost mark, which end the lifetimes of the buffers allocated
    since, newest first. Returns the sizes, lifetimes in events and the bump offsets."""
    rng = np.random.default_rng(seed)
    off, t = 0, 0
    recs, live, marks = [], [], []
    for _ in range(n_ops):
        r = rng.random()
        if r < 0.55 or not live:
            nb = int(np.exp(rng.uniform(np.log(64), np.log(256 << 20))))
            a = (off + ALIGN - 1) // ALIGN * ALIGN
            off = a + nb
            recs.append([nb, t, None, a])
            live.append(len(recs) - 1)
            t += 1
        elif r < 0.75:
            marks.append((off, len(live)))
        elif marks:
            m, k = marks.pop()
            off = m
            for i in reversed(live[k:]):
                recs[i][2] = t
                t += 1
            del live[k:]
    for i in live:
        recs[i][2] = t
    r = np.array(recs, dtype=np.int64)
    return r[:, 0], r[:, 1], r[:, 2], r[:, 3]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_stack_shaped_sequence_gets_the_bump_offsets(place, seed):
    nbytes, t0, t1, bump = stack_sequence(seed)
    assert len(nbytes) > 1000
    peak, off = place(nbytes, t0, t1)
    assert np.array_equal(off, bump)
    assert peak == int((bump + nbytes).max())


def test_bad_input_is_refused(place):
    assert place([1024], [3], [3])[0] < 0                     # empty lifetime
    assert place([1024], [3], [2])[0] < 0
    assert place([-1], [0], [1])[0] < 0
    assert place([1024], [0], [1], placement=2)[0] < 0
    assert place([], [], [])[0] == 0
