"""CPU: frame launches into a tile set on the host side - tw_tile_set_create_tiles_launch and tw_tile_set_stale_after are exported and listed in ABI_SYMBOLS,
the ctypes mirror of tw_tile_set_frame matches the header, null arguments are refused without a device, and the stale_after rules of csrc/tw_tileset_rules.h
(remove, then put, then stale) agree with a Python model on random sets."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_tile_set_host import _layout, _model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("tw_tile_set_create_tiles_launch", "tw_tile_set_stale_after")


def test_entry_points_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for name in NAMES:
        assert " T %s\n" % name in out
        assert name in tw.ABI_SYMBOLS


def test_mirror_matches_the_header(tw, tmp_path):
    _layout(tmp_path, "tw_tile_set_frame", tw.TileSetFrame)


def test_null_arguments_without_a_device(tw):
    L = tw.lib
    xy = (C.c_int32 * 2)(0, 0)
    sp = tw.ShadowParams()
    k = C.c_uint32()
    frame = tw.TileSetFrame(None, 0, C.cast(xy, C.c_void_p), None, None)
    outs = tw.TileOutputs()
    assert L.tw_tile_set_create_tiles_launch(None, None, C.cast(xy, C.c_void_p), 1, 64, 64, 0.1, 0.1, None, 0, None, 0.0, 0.0, 0, C.byref(outs), None,
                                             C.byref(frame)) == tw.TW_ERR_ARG
    assert L.tw_tile_set_stale_after(None, C.byref(sp), 1, None, 0, C.cast(xy, C.c_void_p), 1, None, 0, C.byref(k)) == tw.TW_ERR_ARG


DRIVER = r"""
#include "tw_tileset_rules.h"
#include <cstdio>
// stdin: R resident pairs (tile i at slot 2i; the odd slots below 2R are free), NL slots with sx sy each, then per slot the 2R valid bits, Q reset flags,
// the removed pairs, the put pairs (each list preceded by its count). stdout: the stale_after pairs.
int main() {
	int R, NL, Q, nr, np;
	twts::state st;
	if (scanf("%d", &R) != 1) return 1;
	for (int i = 0; i < R; ++i) {twts::key k; if (scanf("%d %d", &k.first, &k.second) != 2) return 1; st.where[k] = 2u*i; st.free_slots.push_back(2u*i + 1);}
	st.used = 2u*R;
	if (scanf("%d", &NL) != 1) return 1;
	std::vector<twts::signs> sg(NL);
	for (auto &s : sg) {if (scanf("%d %d", &s.sx, &s.sy) != 2) return 1;}
	st.valid.assign(NL, std::vector<uint8_t>(2*R));
	for (auto &v : st.valid) {for (auto &b : v) {int x; if (scanf("%d", &x) != 1) return 1; b = (uint8_t)x;}}
	if (scanf("%d", &Q) != 1) return 1;
	std::vector<uint8_t> reset(Q);
	for (auto &r : reset) {int x; if (scanf("%d", &x) != 1) return 1; r = (uint8_t)x;}
	if (scanf("%d", &nr) != 1) return 1;
	std::vector<twts::key> rk(nr);
	for (auto &k : rk) {if (scanf("%d %d", &k.first, &k.second) != 2) return 1;}
	if (scanf("%d", &np) != 1) return 1;
	std::vector<twts::key> pk(np);
	for (auto &k : pk) {if (scanf("%d %d", &k.first, &k.second) != 2) return 1;}
	twts::state const before = st;
	for (auto const &k : twts::stale_after(st, rk, pk, sg, reset)) printf("%d %d\n", k.first, k.second);
	return (before.where == st.where && before.valid == st.valid) ? 0 : 3;   // the argument is a copy: the state stays as it was
}
"""


def _downstream(res, seeds, sx, sy):
    out, todo = set(), list(seeds)
    while todo:
        k = todo.pop()
        if k in res and k not in out:
            out.add(k)
            todo += [(k[0] - sx, k[1]), (k[0], k[1] - sy)]
    return out


def _stale_after_model(res, signs, valid, reset, removed, put):
    """valid: per slot {key: bit}. Remove, then put, then the resident tiles stale for one of the len(reset) asked slots, in (x, y) order."""
    res, valid = set(res), [dict(v) for v in valid]
    res -= set(removed)
    for v, (sx, sy) in zip(valid, signs):
        for k in removed:
            del v[k]
        seeds = [s for k in removed for s in ((k[0] - sx, k[1]), (k[0], k[1] - sy))]
        for k in _downstream(res, seeds, sx, sy):
            v[k] = 0
    res |= set(put)
    for v, (sx, sy) in zip(valid, signs):
        for k in _downstream(res, put, sx, sy):
            v[k] = 0
    return sorted(k for k in res if any(reset[l] or not valid[l][k] for l in range(len(reset))))


@pytest.fixture(scope="module")
def rules_exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("frame_rules")
    (d / "driver.cpp").write_text(DRIVER)
    exe = str(d / "driver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "3dworld_b200", "csrc"), str(d / "driver.cpp"), "-o", exe])
    return exe


@pytest.mark.parametrize("seed", range(40))
def test_stale_after_matches_the_model(rules_exe, seed):
    rng = np.random.default_rng(1000 + seed)
    w, h = int(rng.integers(1, 9)), int(rng.integers(1, 9))
    cells = [(x - 2, y - 1) for y in range(h + 2) for x in range(w + 2)]
    res = [c for c in cells if rng.random() < 0.6] or cells[:1]
    nl = int(rng.integers(1, 3))
    signs = [(int(rng.choice([-1, 1])), int(rng.choice([-1, 1]))) for _ in range(nl)]
    valid = []
    for sx, sy in signs:                                      # invalidity closed downstream in every slot, as the set keeps it
        v = [int(b) for b in rng.random(len(res)) < 0.8]
        v, _ = _model(res, sx, sy, [k for k, b in zip(res, v) if not b], v, [])
        valid.append(v)
    reset = [int(rng.random() < 0.15) for _ in range(int(rng.integers(1, nl + 1)))]
    removed = [res[int(i)] for i in rng.choice(len(res), int(rng.integers(0, min(4, len(res)) + 1)), replace=False)]
    free = [c for c in cells if c not in removed]
    put = [free[int(i)] for i in rng.choice(len(free), int(rng.integers(0, min(6, len(free)) + 1)), replace=False)]
    bits = []
    for v in valid:                                           # slot 2i holds tile i; the free odd slots hold stale bits that a reuse must not keep
        row = []
        for b in v:
            row += [b, int(rng.integers(0, 2))]
        bits.append(row)
    inp = "%d\n%s\n%d\n%s\n%s\n%d\n%s\n%d\n%s\n%d\n%s\n" % (
        len(res), "\n".join("%d %d" % k for k in res), nl, "\n".join("%d %d" % s for s in signs), "\n".join(" ".join(map(str, r)) for r in bits),
        len(reset), " ".join(map(str, reset)), len(removed), "\n".join("%d %d" % k for k in removed), len(put), "\n".join("%d %d" % k for k in put))
    r = subprocess.run([rules_exe], input=inp, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [tuple(int(v) for v in line.split()) for line in r.stdout.split("\n") if line.strip()]
    expect = _stale_after_model(res, signs, [dict(zip(res, v)) for v in valid], reset, removed, put)
    assert got == expect
    # with no removes and puts it is tw_tile_set_stale's rule
    if not removed and not put:
        assert got == sorted(k for k in res if any(reset[l] or not dict(zip(res, valid[l]))[k] for l in range(len(reset))))
