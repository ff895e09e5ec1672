"""CPU: tile sets on the host side - the entry points are exported and listed in ABI_SYMBOLS, the ctypes mirrors of tw_tile_set_light / tw_tile_set_request
match the header, null arguments are refused without a device, the C++ adapter's tw3d::tile_set compiles against the library, and the cache rules of
csrc/tw_tileset_rules.h (downstream invalidation, the recompute batch) agree with a Python model on random sets."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("tw_tile_set_create", "tw_tile_set_destroy", "tw_tile_set_put", "tw_tile_set_remove", "tw_tile_set_stale", "tw_tile_set_shadows_launch")


def test_entry_points_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for name in NAMES:
        assert " T %s\n" % name in out
        assert name in tw.ABI_SYMBOLS
    assert tw.lib.tw_abi_version() == 1


def _layout(tmp_path, ctype, cls):
    src = tmp_path / ("%s.c" % ctype)
    fields = [f for f, _ in cls._fields_]
    src.write_text("#include <tw3d.h>\n#include <stdio.h>\n#include <stddef.h>\nint main(void) {printf(\"%%zu\", sizeof(%s));" % ctype +
                   "".join('printf(" %%zu", offsetof(%s, %s));' % (ctype, f) for f in fields) + "return 0;}\n")
    exe = str(tmp_path / ctype)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    nums = [int(v) for v in subprocess.check_output([exe], text=True).split()]
    assert nums[0] == C.sizeof(cls)
    assert nums[1:] == [getattr(cls, f).offset for f in fields]


def test_mirrors_match_the_header(tw, tmp_path):
    _layout(tmp_path, "tw_tile_set_light", tw.TileSetLight)
    _layout(tmp_path, "tw_tile_set_request", tw.TileSetRequest)


def test_null_arguments_without_a_device(tw):
    L = tw.lib
    h = C.c_void_p()
    xy = (C.c_int32 * 2)(0, 0)
    z = (C.c_float * 4)()
    sp = tw.ShadowParams()
    k = C.c_uint32()
    assert L.tw_tile_set_create(None, 4, 1, C.byref(h)) == tw.TW_ERR_ARG and not h.value
    assert L.tw_tile_set_put(None, C.cast(xy, C.c_void_p), 1, C.cast(z, C.c_void_p)) == tw.TW_ERR_ARG
    assert L.tw_tile_set_remove(None, C.cast(xy, C.c_void_p), 1) == tw.TW_ERR_ARG
    assert L.tw_tile_set_stale(None, C.byref(sp), 1, None, 0, C.byref(k)) == tw.TW_ERR_ARG
    assert L.tw_tile_set_shadows_launch(None, C.byref(tw.TileSetRequest())) == tw.TW_ERR_ARG
    L.tw_tile_set_destroy(None)                               # a no-op


def test_adapter_tile_set_compiles(tw, tmp_path):
    from test_cpp_tile_set import build_exe
    assert os.access(build_exe(tw, tmp_path), os.X_OK)


# ---- the cache rules against a model ----
DRIVER = r"""
#include "tw_tileset_rules.h"
#include <cstdio>
// stdin: R pairs (resident), sx sy, S seed pairs, the valid bit of each resident tile, Q requested pairs
// stdout: the valid bits after invalidate_downstream(seeds), then the recompute batch for the requested tiles on those bits
int main() {
	int R, sx, sy, S, Q;
	twts::index_map where;
	if (scanf("%d", &R) != 1) return 1;
	std::vector<twts::key> res(R);
	for (int i = 0; i < R; ++i) {if (scanf("%d %d", &res[i].first, &res[i].second) != 2) return 1; where[res[i]] = (uint32_t)i;}
	if (scanf("%d %d %d", &sx, &sy, &S) != 3) return 1;
	std::vector<twts::key> seeds(S);
	for (auto &k : seeds) {if (scanf("%d %d", &k.first, &k.second) != 2) return 1;}
	std::vector<uint8_t> valid(R + 3, 1);                    // slots past the resident ones stay untouched
	for (int i = 0; i < R; ++i) {int v; if (scanf("%d", &v) != 1) return 1; valid[i] = (uint8_t)v;}
	if (scanf("%d", &Q) != 1) return 1;
	std::vector<twts::key> req(Q);
	for (auto &k : req) {if (scanf("%d %d", &k.first, &k.second) != 2) return 1;}
	twts::invalidate_downstream(where, seeds, sx, sy, valid);
	for (int i = 0; i < R; ++i) printf("%d ", (int)valid[i]);
	printf("\n%d %d %d\n", (int)valid[R], (int)valid[R + 1], (int)valid[R + 2]);
	for (auto const &k : twts::recompute_batch(where, valid, req, sx, sy)) printf("%d %d\n", k.first, k.second);
	return 0;
}
"""


def _model(res, sx, sy, seeds, valid, req):
    where = {k: i for i, k in enumerate(res)}
    valid = list(valid)
    todo, seen = list(seeds), set()
    while todo:                                               # downstream: the tiles whose incoming rows come from k
        k = todo.pop()
        if k not in where or k in seen:
            continue
        seen.add(k)
        valid[where[k]] = 0
        todo += [(k[0] - sx, k[1]), (k[0], k[1] - sy)]
    batch, todo = set(), [k for k in req]
    while todo:                                               # upstream of the invalid requested tiles, through invalid tiles only
        k = todo.pop()
        if k not in where or k in batch or valid[where[k]]:
            continue
        batch.add(k)
        todo += [(k[0] + sx, k[1]), (k[0], k[1] + sy)]
    return valid, batch


@pytest.fixture(scope="module")
def rules_exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("rules")
    (d / "driver.cpp").write_text(DRIVER)
    exe = str(d / "driver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "3dworld_b200", "csrc"), str(d / "driver.cpp"), "-o", exe])
    return exe


@pytest.mark.parametrize("seed", range(40))
def test_closure_rules_match_the_model(rules_exe, seed):
    rng = np.random.default_rng(seed)
    w, h = int(rng.integers(1, 9)), int(rng.integers(1, 9))
    cells = [(x - 3, y + 2) for y in range(h) for x in range(w)]
    res = [c for c in cells if rng.random() < 0.75] or cells[:1]          # holes: the walks stop at tiles that are not resident
    sx, sy = int(rng.choice([-1, 1])), int(rng.choice([-1, 1]))
    seeds = [cells[int(i)] for i in rng.integers(0, len(cells), int(rng.integers(0, 4)))] + [(99, 99)]
    valid = [int(v) for v in rng.random(len(res)) < 0.8]
    # the model's invariant: invalidity is closed downstream (what the set maintains)
    valid, _ = _model(res, sx, sy, [k for k, v in zip(res, valid) if not v], valid, [])
    req = [res[int(i)] for i in rng.choice(len(res), int(rng.integers(1, len(res) + 1)), replace=False)]
    inp = "%d\n%s\n%d %d %d\n%s\n%s\n%d\n%s\n" % (len(res), "\n".join("%d %d" % k for k in res), sx, sy, len(seeds), "\n".join("%d %d" % k for k in seeds),
                                                 " ".join(map(str, valid)), len(req), "\n".join("%d %d" % k for k in req))
    out = subprocess.run([rules_exe], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
    mv, mb = _model(res, sx, sy, seeds, valid, req)
    assert [int(v) for v in out[0].split()] == mv
    assert out[1].split() == ["1", "1", "1"]
    got = [tuple(int(v) for v in line.split()) for line in out[2:] if line.strip()]
    assert len(got) == len(set(got)) and set(got) == mb
    # a valid tile never depends on an invalid one: nothing upstream of a valid tile is in the batch
    where = {k: i for i, k in enumerate(res)}
    for k in mb:
        for d in ((k[0] - sx, k[1]), (k[0], k[1] - sy)):
            assert d not in where or not mv[where[d]]
