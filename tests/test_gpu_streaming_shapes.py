"""GPU: the streaming passes (16-bit heightmap pack from_floats_u16 / unpack to_floats_u16, min/max) at the sizes where their grid-stride loops take a
second pass, on device views that are not 16-byte (input) or 8-byte (output) aligned, at the edges of the pack range and on every 16-bit code; bit for bit
against the plain-C oracle (numpy for min/max).

from_floats launches at most T = 16*SMs blocks' worth of threads (256 per block) and each thread of the aligned branch packs 4 values, so the aligned
branch wraps above 4T values and the unaligned one above T; min/max launches 8*SMs blocks and wraps far earlier, so for it the new cases are the offsets
and an extreme value at the first or last index."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NAN = float("nan")
MULT, ADD = 0.0123, -1.5


@pytest.fixture(scope="module")
def T():
    import torch
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count * 256


def _values(n, seed):
    """n heights whose packed value (h - ADD)/MULT covers [0, 256) and includes both ends of the range."""
    v = np.random.default_rng(seed).uniform(ADD, ADD + 255.99 * MULT, n).astype(np.float32)
    v[0] = np.float32(ADD)
    if n > 1:
        v[-1] = _below_256()
    return v


def _packed(h):
    """(h - add)*float(1/mult) in fp32, as heightmap_t::from_floats computes it (src/heightmap.cpp:206-210)."""
    div = np.float32(1.0 / np.float64(np.float32(MULT)))
    return np.float32(np.float32(np.float32(h) - np.float32(ADD)) * div)


def _below_256():
    """The largest height that packs to a value below 256."""
    h = np.float32(ADD + 256.0 * MULT)
    while _packed(np.nextafter(h, np.float32(np.inf))) < 256.0:
        h = np.nextafter(h, np.float32(np.inf))
    while not _packed(h) < 256.0:
        h = np.nextafter(h, np.float32(-np.inf))
    return h


def _sizes(T):
    return [T - 1, T, T + 1] + [4 * T + k for k in range(5)]


def _view(t, off, n):
    """Elements off..off+n of a 1-D CUDA tensor: a contiguous view whose address is off elements past the allocation's (256-byte aligned) start."""
    return t[off:off + n]


def _cuda(a):
    import torch
    t = torch.from_numpy(a).cuda()
    torch.cuda.synchronize()
    return t


def test_pack_sizes(oracle, ctx, T):
    """Host input (staged into aligned scratch: the aligned branch) around T and 4T, plus the 8192^2 heightmap."""
    for n in _sizes(T) + [8192 * 8192]:
        v = _values(n, n)
        exp, bad = oracle.from_floats_u16(v, MULT, ADD)
        assert bad == 0
        got = ctx.from_floats_u16(v, MULT, ADD)
        assert np.array_equal(got, exp), n
        back = ctx.to_floats_u16(got, MULT, ADD)
        assert np.array_equal(back.view(np.uint32), oracle.to_floats_u16(exp, MULT, ADD).view(np.uint32)), n


def test_pack_unaligned_views(oracle, ctx, T):
    """Input views 1-3 floats and output views 1-3 uint16 past an aligned address run the unaligned branch; offset 4 of both is aligned again."""
    import torch
    for n in (T - 1, T + 1, 4 * T + 3):
        v = _values(n, 7 * n)
        exp, _ = oracle.from_floats_u16(v, MULT, ADD)
        src = torch.zeros(n + 8, dtype=torch.float32, device="cuda")
        for off_in, off_out in ((1, 0), (2, 0), (3, 0), (0, 1), (0, 2), (0, 3), (3, 1), (4, 4)):
            src[off_in:off_in + n].copy_(torch.from_numpy(v))
            dst = torch.full((2 * (n + 8),), 0xAB, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            ctx.from_floats_u16(_view(src, off_in, n), MULT, ADD, out=_view(dst, 2 * off_out, 2 * n))
            got = dst.cpu().numpy()
            assert np.array_equal(got[2 * off_out:2 * (off_out + n)], exp), (n, off_in, off_out)
            assert (got[:2 * off_out] == 0xAB).all() and (got[2 * (off_out + n):] == 0xAB).all()


def test_unpack_unaligned_views(oracle, ctx, T):
    """to_floats from uint16 views 1-3 codes past an aligned address into float views 1-3 past one."""
    import torch
    for n in (T - 1, T + 1, 4 * T + 3):
        data = np.random.default_rng(n).integers(0, 256, 2 * n, dtype=np.uint8)
        exp = oracle.to_floats_u16(data, MULT, ADD)
        src = torch.zeros(2 * (n + 8), dtype=torch.uint8, device="cuda")
        for off_in, off_out in ((1, 0), (2, 1), (3, 2), (0, 3)):
            src[2 * off_in:2 * (off_in + n)].copy_(torch.from_numpy(data))
            dst = torch.full((n + 8,), NAN, dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            ctx.to_floats_u16(_view(src, 2 * off_in, 2 * n), MULT, ADD, out=_view(dst, off_out, n))
            got = dst.cpu().numpy()
            assert np.array_equal(got[off_out:off_out + n].view(np.uint32), exp.view(np.uint32)), (n, off_in, off_out)
            assert np.isnan(got[:off_out]).all() and np.isnan(got[off_out + n:]).all()


def test_unpack_every_code(oracle, ctx):
    """All 65536 codes, against a float64 restatement of heightmap_t::to_floats (src/heightmap.cpp:199) and the oracle."""
    codes = np.arange(65536, dtype=np.uint16)
    data = codes.view(np.uint8)                       # little endian: data[2i] = low byte (fraction), data[2i+1] = high byte
    v = (np.float64(1.0) * (codes & 0xff) / 256.0 + (codes >> 8)).astype(np.float32)
    for mult, add in ((MULT, ADD), (1.0, 0.0), (-3.7, 1.0e4), (1.0e-7, 0.25)):
        exp = np.float32(mult) * v + np.float32(add)
        got = ctx.to_floats_u16(data, mult, add)
        assert np.array_equal(got.view(np.uint32), exp.view(np.uint32)), (mult, add)
        assert np.array_equal(got.view(np.uint32), oracle.to_floats_u16(data, mult, add).view(np.uint32))


def test_pack_range_edges(oracle, ctx):
    """v = 0 packs to 0 and the largest v below 256 to 0xffff; both ends of every size of tail."""
    for n in (1, 2, 3, 4, 5, 7):
        v = np.full(n, _below_256(), np.float32)
        v[::2] = np.float32(ADD)
        exp, bad = oracle.from_floats_u16(v, MULT, ADD)
        assert bad == 0 and exp.view(np.uint16)[0] == 0
        got = ctx.from_floats_u16(v, MULT, ADD)
        assert np.array_equal(got, exp)
    assert ctx.from_floats_u16(np.array([_below_256()], np.float32), MULT, ADD).view(np.uint16)[0] == 0xffff


BAD = {"nan": lambda: np.float32(NAN), "inf": lambda: np.float32(np.inf), "-inf": lambda: np.float32(-np.inf),
       "just below 0": lambda: np.nextafter(np.float32(ADD), np.float32(-np.inf)), "-1": lambda: np.float32(ADD - MULT),
       "256": lambda: np.nextafter(_below_256(), np.float32(np.inf)), "300": lambda: np.float32(ADD + 300.0 * MULT)}


@pytest.mark.parametrize("bad", sorted(BAD))
def test_pack_bad_values(tw, oracle, ctx, T, bad):
    """NaN, +-inf, v < 0 and v >= 256 are TW_ERR_ARG at index 0, in the aligned branch's second grid-stride pass and its tail loop, and in the unaligned
    branch."""
    import torch
    n = 4 * T + 5                                     # T + 1 float4 groups: the aligned loop wraps once, then a tail of 1
    v = _values(n, 3)
    for where, ix, off in (("first", 0, 0), ("second pass", 4 * T + 1, 0), ("tail", n - 1, 0), ("unaligned", n // 2, 1), ("unaligned last", n - 1, 3)):
        w = v.copy()
        w[ix] = BAD[bad]()
        assert oracle.from_floats_u16(w, MULT, ADD)[1] == 1
        src = torch.zeros(n + 4, dtype=torch.float32, device="cuda")
        src[off:off + n].copy_(torch.from_numpy(w))
        torch.cuda.synchronize()
        with pytest.raises(tw.TwError) as e:
            ctx.from_floats_u16(_view(src, off, n) if off else w, MULT, ADD)
        assert e.value.status == tw.TW_ERR_ARG, where


def test_minmax_sizes_and_views(ctx, T):
    import torch
    for n in _sizes(T):
        v = np.random.default_rng(n).standard_normal(n).astype(np.float32)
        for ix in (0, n - 1):
            for ext in (np.float32(-1.0e30), np.float32(1.0e30)):
                w = v.copy()
                w[ix] = ext
                assert ctx.minmax(w) == (float(w.min()), float(w.max())), (n, ix)
        src = torch.zeros(n + 4, dtype=torch.float32, device="cuda")
        for off in (1, 2, 3):
            w = v.copy()
            w[0], w[-1] = np.float32(-7.0), np.float32(9.0)
            src.fill_(0.0)
            src[off:off + n].copy_(torch.from_numpy(w))
            src[:off].fill_(-100.0)
            src[off + n:].fill_(100.0)
            torch.cuda.synchronize()
            assert ctx.minmax(_view(src, off, n)) == (-7.0, 9.0), (n, off)
