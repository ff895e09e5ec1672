"""CPU: the domain-warp simplex kernel's hash table holds gradient-table byte offsets (csrc/tw_noise2.cuh, simplex_hash_entry) instead of
hash values. This rebuilds that table in numpy fp32 (the offsets are denormals; numpy keeps them, as the kernel does without -ftz) and checks,
for every reachable (ix, iy, i1.y), that the three addresses the kernel forms from it are bit for bit the addresses lut_offsets() gives the
second-permute arguments the reference computes: permute(iy + {0, i1.y, 1}) + ix + {0, i1.x, 1}."""
import numpy as np

f32 = np.float32
ENTRY = 128                                   # bytes per gradient entry in the 8-copy layout (LUT_ENTRY_BYTES)


def permute(x):
    v = (x * f32(34.0) + f32(1.0)) * x
    return v - np.floor(v * (f32(1.0) / f32(289.0))) * f32(289.0)


def bits(v):
    """The float whose bit pattern is the non-negative integer v"""
    return np.asarray(v, np.int64).astype(np.uint32).view(f32)


def test_hash_entries_give_the_gradient_offsets():
    k = np.arange(291, dtype=f32)                                     # SIMPLEX_HASH_N entries
    p0, p1 = permute(k).astype(np.int64), permute(k + f32(1.0)).astype(np.int64)
    table = np.stack([bits(ENTRY * p0), bits(ENTRY * (p0 + 1)), bits(ENTRY * (p1 + 1)), bits(0 * p0)], axis=1)
    assert table.dtype == f32 and np.all(table < np.finfo(f32).tiny)  # every entry is a denormal (or zero)
    ix, iy = np.meshgrid(np.arange(290, dtype=f32), np.arange(290, dtype=f32), indexing="ij")   # mod_int289_lazy: 0 .. 289
    ix, iy = ix.ravel(), iy.ravel()
    j = iy.astype(np.int64)
    d128 = bits(ENTRY)
    for Lb in (0, 7 * 16, (1 << 18) - 1 - 7 * 16):                 # the lane's copy of entry 0: a shared-memory address below 2^18
        Lbf = bits(Lb)
        bx = ix * d128 + Lbf                                          # lut_offsets(ix): exact product, exact sum
        for i1y in (f32(0.0), f32(1.0)):
            i1x = f32(1.0) - i1y
            k0 = table[j, 0] + bx
            k1 = (table[j + 1, 0] if i1y else table[j, 1]) + bx        # the word at entry iy's address + 4 + (pitch - 4)*i1.y
            k2 = table[j, 2] + bx
            q0, q1, q2 = permute(iy), permute(iy + i1y), permute(iy + f32(1.0))
            for got, arg in ((k0, q0 + ix), (k1, (q1 + ix) + i1x), (k2, (q2 + ix) + f32(1.0))):
                want = arg * d128 + Lbf                               # the parent's lut_offsets(p)
                assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
                assert np.array_equal(got.view(np.uint32).astype(np.int64), ENTRY * arg.astype(np.int64) + Lb)
    assert ENTRY * 578 + (1 << 18) < 1 << 19                          # the largest address stays far inside the denormal range (2^23)
