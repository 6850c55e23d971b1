"""CPU-only: implicit_b200.pcg64 follows numpy's PCG64 float32 stream exactly (the state dict numpy leaves after a draw,
which random_state kinds fit() draws on the device), and a restatement of fill_pcg64_kernel's thread-to-stream mapping
(csrc/gen.cu) gives numpy's draw bit for bit."""
import numpy as np
import pytest

from implicit_b200 import pcg64
from implicit_b200.utils import check_random_state


def full_state(gen):
    return gen.bit_generator.state


def with_buffered_half(seed):
    """A Generator whose state holds a buffered high half (has_uint32 = 1)."""
    g = np.random.default_rng(seed)
    g.random(1, dtype=np.float32)
    assert g.bit_generator.state["has_uint32"] == 1
    return g


@pytest.mark.parametrize("has", [0, 1])
@pytest.mark.parametrize("shape", [(n,) for n in range(10)] + [(3, 5), (4, 1), (1, 7), (0, 64), (5, 0), (17, 65)])
def test_state_after_draws_matches_numpy(has, shape):
    g = with_buffered_half(11) if has else np.random.default_rng(11)
    want = pcg64.after_float32_draws(pcg64.get_state(g), int(np.prod(shape)))
    before = pcg64.get_state(g)
    g.random(shape, dtype=np.float32)
    assert pcg64.get_state(g) == want
    if np.prod(shape) == 0:
        assert pcg64.get_state(g) == before


@pytest.mark.parametrize("has", [0, 1])
@pytest.mark.parametrize("users,items,f", [(1, 1, 1), (3, 2, 5), (2, 3, 5), (7, 0, 3), (0, 4, 3), (10, 13, 64)])
def test_user_then_item_sequence(has, users, items, f):
    g = with_buffered_half(5) if has else np.random.default_rng(5)
    st = pcg64.get_state(g)
    st = pcg64.after_float32_draws(st, users * f)
    st = pcg64.after_float32_draws(st, items * f)
    g.random((users, f), dtype=np.float32)
    g.random((items, f), dtype=np.float32)
    assert pcg64.get_state(g) == st
    # written back, the state is numpy's whole dict
    h = np.random.default_rng(99)
    pcg64.set_state(h, st)
    assert full_state(h) == full_state(g)
    assert np.array_equal(h.random(9, dtype=np.float32), g.random(9, dtype=np.float32))


@pytest.mark.parametrize("has", [0, 1])
@pytest.mark.parametrize("n", [2**32 + 1, 2**33, 65 * 2**26 + 3, 2**40 + 7, 10**15])
def test_huge_counts_against_numpy_advance(has, n):
    g = with_buffered_half(3) if has else np.random.default_rng(3)
    s, inc, h, u = pcg64.get_state(g)
    got = pcg64.after_float32_draws((s, inc, h, u), n)
    steps = (n - h + 1) // 2
    adv = np.random.Generator(np.random.PCG64())
    pcg64.set_state(adv, (s, inc, 0, 0))
    adv.bit_generator.advance(steps)
    assert got[0] == adv.bit_generator.state["state"]["state"]
    assert got[1] == inc and got[2] == (n - h) % 2
    # uinteger: the high half of the last step's output, as numpy leaves it after the step's two halves
    last = np.random.Generator(np.random.PCG64())
    pcg64.set_state(last, (pcg64.advance(s, inc, steps - 1), inc, 0, 0))
    last.random(2, dtype=np.float32)
    assert got[3] == last.bit_generator.state["uinteger"]
    assert pcg64.get_state(last)[0] == got[0]


def test_advance_is_numpys():
    g = np.random.default_rng(8)
    s, inc, _, _ = pcg64.get_state(g)
    for k in (0, 1, 2, 3, 1000, 2**64 + 5):
        a = np.random.Generator(np.random.PCG64())
        pcg64.set_state(a, (s, inc, 0, 0))
        a.bit_generator.advance(k)
        assert pcg64.advance(s, inc, k) == a.bit_generator.state["state"]["state"]


@pytest.mark.parametrize("kind,device", [
    ("none", True), ("int", True), ("seedsequence", True), ("randomstate", True), ("pcg64", True),
    ("pcg64-bitgen", True), ("pcg64dxsm", False), ("philox", False), ("mt19937", False), ("sfc64", False)])
def test_routing(kind, device):
    rs = {"none": None, "int": 7, "seedsequence": np.random.SeedSequence(7),
          "randomstate": np.random.RandomState(7), "pcg64": np.random.default_rng(7),
          "pcg64-bitgen": np.random.PCG64(7), "pcg64dxsm": np.random.Generator(np.random.PCG64DXSM(7)),
          "philox": np.random.Generator(np.random.Philox(7)), "mt19937": np.random.Generator(np.random.MT19937(7)),
          "sfc64": np.random.Generator(np.random.SFC64(7))}[kind]
    assert pcg64.device_drawable(check_random_state(rs)) is device


def test_generator_at():
    g = with_buffered_half(21)
    st = pcg64.get_state(g)
    h = pcg64.generator_at(st)
    assert full_state(h) == full_state(g)
    assert np.array_equal(h.random((4, 3), dtype=np.float32), g.random((4, 3), dtype=np.float32))


# ----------------------------------------------------------------------------- the kernel's mapping, restated
def kernel_fill(state, rows, f, ld, scale, threads, draws, grid):
    """fill_pcg64_kernel and its launcher (csrc/gen.cu) at a block of `threads` threads, `draws` 64-bit draws per thread
    and tile, and `grid` blocks, restated in Python ints: the jump table, the grid stride, each thread's run, the
    shared-memory tile and the write-out through fdiv."""
    s0, inc, has, u0 = state
    mask = (1 << 128) - 1
    x = np.zeros((rows, ld), dtype=np.float32)
    n = rows * f
    if n == 0:
        return x
    tile_n = threads * draws * 2
    first = 1 if has else 0
    m = n - first
    mult, plus = [], []
    a, c = pcg64.MULT, inc
    for _ in range(64):
        mult.append(a)
        plus.append(c)
        c = (a + 1) * c & mask
        a = a * a & mask

    def jump(s, k):
        j = 0
        while k:
            if k & 1:
                s = (mult[j] * s + plus[j]) & mask
            j += 1
            k >>= 1
        return s

    sm, sp = 1, 0  # the composed map of grid * tile_n / 2 draws
    k, j = grid * (tile_n // 2), 0
    while k:
        if k & 1:
            sm, sp = mult[j] * sm & mask, (mult[j] * sp + plus[j]) & mask
        j += 1
        k >>= 1
    fdiv = 0 if f == 1 else ((1 << 32) + f - 1) // f

    def value(u32):
        return np.float32(np.float32(u32 >> 8) * np.float32(2.0 ** -24)) * np.float32(scale)

    flat = x.reshape(-1)
    if first:
        flat[0] = value(u0)
    tiles = (m + tile_n - 1) // tile_n
    for b in range(grid):
        start = [jump(s0, b * (tile_n // 2) + t * draws) for t in range(threads)]
        for tt in range(b, tiles, grid):
            p0 = tt * tile_n
            smem = np.full(tile_n, np.nan, dtype=np.float32)
            for t in range(threads):
                if p0 + t * 2 * draws < m:
                    s = start[t]
                    for d in range(draws):
                        s = (s * pcg64.MULT + inc) & mask
                        v = pcg64.output(s)
                        smem[t * 2 * draws + 2 * d] = value(v & 0xFFFFFFFF)
                        smem[t * 2 * draws + 2 * d + 1] = value(v >> 32)
                start[t] = (sm * start[t] + sp) & mask
            e0 = p0 + first
            r0, c0 = e0 // f, e0 % f
            for l in range(min(tile_n, m - p0)):
                cc = c0 + l
                q = cc if f == 1 else (cc * fdiv) >> 32
                flat[(r0 + q) * ld + (cc - q * f)] = smem[l]
    return x


@pytest.mark.parametrize("has", [0, 1])
@pytest.mark.parametrize("rows,f,ld,threads,draws,grid", [
    (7, 5, 16, 4, 3, 2),      # 24-value tiles end mid-row
    (13, 3, 16, 2, 5, 3),     # more tiles than blocks: grid-stride steps
    (1, 1, 16, 1, 1, 1), (2, 1, 16, 3, 2, 1), (5, 17, 32, 4, 4, 5), (9, 7, 16, 3, 3, 4), (3, 33, 48, 2, 7, 2)])
def test_kernel_mapping_is_numpys_draw(has, rows, f, ld, threads, draws, grid):
    g = with_buffered_half(1234) if has else np.random.default_rng(1234)
    st = pcg64.get_state(g)
    got = kernel_fill(st, rows, f, ld, 0.01, threads, draws, grid)
    want = g.random((rows, f), dtype=np.float32) * np.float32(0.01)
    assert np.array_equal(got[:, :f].view(np.uint32), want.view(np.uint32))
    assert not got[:, f:].any()
    assert pcg64.get_state(g) == pcg64.after_float32_draws(st, rows * f)


def test_fdiv_divides_every_tile_column():
    """__umulhi(c, ceil(2^32 / f)) == c // f for every column offset the kernel forms (c < f + 4096) and every width
    2 <= f <= 1024 (f = 1 takes q = c); the multiplier fits 32 bits."""
    c = np.arange(1024 + 4096, dtype=np.uint64)
    for f in range(2, 1025):
        fdiv = np.uint64(((1 << 32) + f - 1) // f)
        assert fdiv < 2**32
        assert np.array_equal((c * fdiv) >> np.uint64(32), c // np.uint64(f)), f
