"""CPU: the ground-mode mesh job on the host side - tw_gen_mesh_launch is exported and listed in ABI_SYMBOLS, the ctypes mirrors of tw_gen_mesh_job and
tw_gen_mesh_info match the header, a NULL context is refused; a numpy restatement of the job's device z estimate (the probe's max |z| as one integer
maximum of float bits, then zmax_est, set_zvals and water_plane_z) held to the host chain's arithmetic (tw3d::gen_mesh's loop and the library's
tw_water_z_height) on flat, sine-like and noise-like data; and the SASS of the droplet and glaciation kernels beside which the job's variants were added,
against the digests of the build before the job existed."""
import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def test_entry_point_is_exported(tw):
    assert "tw_gen_mesh_launch" in tw.ABI_SYMBOLS and hasattr(tw.lib, "tw_gen_mesh_launch")
    assert tw.lib.tw_abi_version() == 1


@pytest.mark.parametrize("struct,name", [("GenMeshJobArgs", "tw_gen_mesh_job"), ("GenMeshInfo", "tw_gen_mesh_info")])
def test_layout(tw, tmp_path, struct, name):
    S = getattr(tw, struct)
    fields = [f for f, _ in S._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tw3d.h"\nint main(void) {printf("%%zu", sizeof(%s)); ' % name
                   + "".join('printf(" %%zu", offsetof(%s, %s)); ' % (name, f) for f in fields) + "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(S)] + [getattr(S, f).offset for f in fields]


def test_launch_refuses_null_context(tw):
    assert tw.lib.tw_gen_mesh_launch(None, None) == tw.TW_ERR_ARG


def ord_key(v):
    """tw_f2ord: the order-preserving uint encoding of the mesh's min/max reduction."""
    u = np.asarray(v, F).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000).astype(np.uint32)


def ord_val(u):
    u = np.uint32(u)
    return np.array([(u & 0x7fffffff) if (u & 0x80000000) else (~u & 0xffffffff)], np.uint32).view(F)[0]


def device_zvals(mesh, probe, sine_mode, glaciate, custom_exp, water_h_off, water_h_off_rel, prev, tw):
    """gen_mesh_zvals_kernel after probe_absmax_kernel, in numpy: the mesh's min/max through the ordered keys, the probe's largest non-NaN |z| as an integer
    maximum of float bits, then the one thread's arithmetic with wpz from the host (twi_water_rel restated)."""
    fin = mesh[~np.isnan(mesh)]
    zmin, zmax = ord_val(ord_key(fin).min()), ord_val(ord_key(fin).max())
    zmax_est = -zmin if zmax < -zmin else zmax
    if zmax == zmin:
        zmax_est = F(float(zmax_est) + 1.0E-6)
        return dict(zmin=zmin, zmax=zmax, zmax_est=zmax_est, zbottom=F(prev[0]), ztop=F(prev[1]), water_plane_z=F(prev[2]))
    a = np.abs(probe.astype(F))
    a = a[~np.isnan(a)]
    m = np.array([a.view(np.uint32).max() if a.size else 0], np.uint32).view(F)[0]
    zmax_est = m if zmax_est < m else zmax_est
    if not sine_mode:
        zmax_est = F(float(zmax_est) * 1.2)
    zmax_est = F(1.1 * float(zmax_est))
    t = F(F(0.42) + F(water_h_off_rel))
    wpz = max(F(0.0), min(t, F(1.0)))
    if glaciate:
        wpz = F(wpz * wpz * wpz) if custom_exp == 0.0 else F(np.power(wpz, F(custom_exp)))
    wpz_z = F(F(wpz * F(2.0 * float(zmax_est))) - zmax_est) + F(water_h_off)
    return dict(zmin=-zmax_est, zmax=zmax_est, zmax_est=zmax_est, zbottom=zmin, ztop=zmax, water_plane_z=F(wpz_z))


def host_zvals(mesh, probe, sine_mode, glaciate, custom_exp, water_h_off, water_h_off_rel, prev, tw):
    """tw3d::gen_mesh's host arithmetic, loop for loop, with the library's tw_water_z_height."""
    fin = mesh[~np.isnan(mesh)]
    zmin, zmax = F(fin.min()), F(fin.max())
    zmax_est = -zmin if zmax < -zmin else zmax
    if zmax == zmin:
        zmax_est = F(float(zmax_est) + 1.0E-6)
        return dict(zmin=zmin, zmax=zmax, zmax_est=zmax_est, zbottom=F(prev[0]), ztop=F(prev[1]), water_plane_z=F(prev[2]))
    for v in probe.ravel():
        a = F(abs(v))
        zmax_est = a if zmax_est < a else zmax_est
    if not sine_mode:
        zmax_est = F(float(zmax_est) * 1.2)
    zmax_est = F(1.1 * float(zmax_est))
    wpz = F(tw.lib.tw_water_z_height(float(zmax_est), glaciate, custom_exp, water_h_off, water_h_off_rel))
    return dict(zmin=-zmax_est, zmax=zmax_est, zmax_est=zmax_est, zbottom=zmin, ztop=zmax, water_plane_z=wpz)


def cases():
    rng = np.random.default_rng(7)
    x = np.linspace(0, 6.0, 64, dtype=F)
    sine = (F(0.3) * np.sin(x)[:, None] * np.cos(F(1.7) * x)[None, :]).astype(F)
    noise = rng.normal(0.0, 0.8, (64, 64)).astype(F)
    spiky = noise.copy()
    spiky[3, 5], spiky[9, 9] = np.nan, F(-7.5)
    yield "flat", np.zeros((64, 64), F), rng.normal(0, 1, (128, 128)).astype(F), True
    yield "flat_negative", np.full((64, 64), F(-0.25)), rng.normal(0, 1, (128, 128)).astype(F), False
    yield "sine", sine, (F(0.35) * np.sin(rng.uniform(0, 9, (128, 128)))).astype(F), True
    yield "sine_probe_lower", sine, (F(0.01) * np.sin(rng.uniform(0, 9, (128, 128)))).astype(F), True
    yield "noise", noise, rng.normal(0.0, 1.1, (128, 128)).astype(F), False
    yield "noise_nan_probe", spiky, np.where(rng.uniform(size=(128, 128)) < 0.01, np.nan, rng.normal(0.0, 2.0, (128, 128))).astype(F), False
    yield "noise_inf_probe", noise, np.where(rng.uniform(size=(128, 128)) < 0.001, np.inf, rng.normal(0.0, 2.0, (128, 128))).astype(F), False


@pytest.mark.filterwarnings("ignore::RuntimeWarning")                     # the infinite probe makes water_plane_z NaN on both sides
@pytest.mark.parametrize("glaciate,custom_exp,h_off,h_rel", [(1, 0.0, 0.0, 0.0), (0, 0.0, 0.05, -0.03), (1, 2.2, -0.1, 0.2), (1, 0.0, 0.0, 0.7)])
def test_device_zvals_restatement_equals_host_chain(tw, glaciate, custom_exp, h_off, h_rel):
    prev = (0.25, 0.75, -0.125)
    for name, mesh, probe, sine_mode in cases():
        d = device_zvals(mesh, probe, sine_mode, glaciate, custom_exp, h_off, h_rel, prev, tw)
        h = host_zvals(mesh, probe, sine_mode, glaciate, custom_exp, h_off, h_rel, prev, tw)
        for k in h:
            assert F(d[k]).view(np.uint32) == F(h[k]).view(np.uint32), (name, k, d[k], h[k])


# SHA-256 of each kernel's SASS instruction words (the encodings cuobjdump -sass prints) in the build before tw_gen_mesh_launch existed, CUDA 12.9: the job adds
# DEV_E variants of the droplet kernel and a record-reading variant of the glaciation kernel, and the existing instantiations' code must not change with them
SASS_CUDA = "12.9"
SASS_PARENT = {
    "droplet_kernel<1,0,0>": "d85805ead8f2e97e070247659ec0e9fc1f372696cce60eae3a6d02ca82b005ac",
    "droplet_kernel<1,0,1>": "d695c5f83c803f31ae570ddf13c0cf6a8fab2b90882e234288009df90f30489a",
    "droplet_kernel<2,0,0>": "571088a81dd038370dfb9f5ab60ab7a6bdd135a6ccdaf798e8408d7f59163aa0",
    "droplet_kernel<2,0,1>": "eadea7e34d004874e21b261da08457340db544a5cf5394af54eb87bfca5c2f2d",
    "droplet_kernel<4,0,0>": "c9f76e3172e746a15b0312e665a3300766e87c16ec7db01e751328824d87c15e",
    "droplet_kernel<4,0,1>": "a25b2e6f81012140375d887f65900c3232fb5106cc1187f4bdde8e4e85c3f6be",
    "droplet_kernel<8,0,0>": "f2e7a76bbe636e8bb0764a6bd0f812e3a1aeb97737bcac16552ee08f5181fa54",
    "droplet_kernel<8,0,1>": "d88b0e19afab8863ddbae07e8e7df5ff3502d0d3696c7237ad34d868537cf358",
    "droplet_kernel<16,0,0>": "7d7fc47560173fa71428aecd16160ad02061c31e544ebe38b619ba23b8c77dc2",
    "droplet_kernel<16,0,1>": "375fb8eba599a24d08b7b7c6e26e04eddd3ca983984a148286737afceeb821f6",
    "droplet_kernel<32,0,0>": "41b8bbad275758d3687dca789738087328e908a1b4db465c63e83819b5d8efd9",
    "droplet_kernel<32,0,1>": "4076591ab0cfb25d61472444f5418d396d782727ebfff91539ae3d2cf2c0bb5a",
    "droplet_kernel<1,1,0>": "e459fdec5aab354f971d173b024f43234506f25b8a7ceb95011b7497d6caa2a4",
    "droplet_kernel<1,1,1>": "f120126c9d1e4bdce22c0212c72358486730dc051e09fda76efd02084764e1a5",
    "droplet_kernel<2,1,0>": "4e587be6ad6d6c99c9c9e24b6a850c620f1267ae1b70c510f24ee14b9f86fa1f",
    "droplet_kernel<2,1,1>": "9a94fbb583f1e7e09e1ab4afabdca72ddce45cf5b468df2c49aa1398dd331621",
    "droplet_kernel<4,1,0>": "68236c005b88402be7066222bc1d68ebd5ab9e81e6b6e099de0013795fcbb77d",
    "droplet_kernel<4,1,1>": "3cb785851a43d384d9546c4d81514c7b9a9e56b285aa3e4ef96438c8f5fe79bb",
    "droplet_kernel<8,1,0>": "dc643fb5f3395c06de6b0f80f09ec6c2afdbac7074e9fd968ab6ae90a90b9094",
    "droplet_kernel<8,1,1>": "1d1888e7e8b2d7126881b2832f75f257c0d19064740835ca09e636cc2acba5c6",
    "droplet_kernel<16,1,0>": "1dd68eb89dba48dab9887d05a72c1caa059eb70362cde96a500925b117c85248",
    "droplet_kernel<16,1,1>": "be9d28b7188dabea47ea10c5566df2b79db04a9e2ed7b237247b35802215078b",
    "droplet_kernel<32,1,0>": "a2afa87d103c78075f11827c4f7e40e1569512a808fd50c2d33dc4f170547838",
    "droplet_kernel<32,1,1>": "776c88630e82ec5c84ff09a031586cf2a8107ee4651197c895df78069962c8d2",
    "droplet_kernel<1,2,0>": "9162e27bd62908a91ba5781c9d2520158c5f78c206d8658238878bf7a54fd023",
    "droplet_kernel<1,2,1>": "1a3384d67ba9c144fa0c2573d6196a3b28a835c50a20d25dbdd5230cfaebfa52",
    "droplet_kernel<2,2,0>": "4b2265b64f4c5f6798bc85ff0ff3763b96e62e0a79a72fca8ce433fe80181729",
    "droplet_kernel<2,2,1>": "d7313956778324896150dd94c2b3fde4a709de07e0732749fecc8bbd3f054429",
    "droplet_kernel<4,2,0>": "8e48b9fec9c2a436d6d15d422db9849e5a39a1e888fab9d77141de8ebb8a8b7c",
    "droplet_kernel<4,2,1>": "8c71a3268a6c1351a4b5405acecad88383db7a616b45a870992572bc68e8fd17",
    "droplet_kernel<8,2,0>": "f827b4e11a88232498aefef717adfdbd6353bf995bc56f5a165a5b22023d41cc",
    "droplet_kernel<8,2,1>": "1a9382b281d4d10df8c953345b5b7286a0ef7263d170d16605991fddde5779c4",
    "droplet_kernel<16,2,0>": "971dce7af108209ec23a528455fafa428b07045f98775c03d1529acaaad8aa12",
    "droplet_kernel<16,2,1>": "cdaedd348b3c0b44bc0836dfee0524245ad4166f051c7ce4ac5aac41dcef6a7a",
    "droplet_kernel<32,2,0>": "1fbbd3df52a950f464a67979cd95330d1c6c8ec16378d4d662f9a95d64d3cab1",
    "droplet_kernel<32,2,1>": "ef78c8688bd33ee87cd7d37efe6f99c3561c65144d2bc62cf47afc1519b93c54",
    "droplet_kernel<1,3,0>": "5daf645fc3930c02211b77ae4a8dc8ea9ebb28ab0b44601631f090da45610f18",
    "droplet_kernel<1,3,1>": "10350d28561a7358a52517539f1d31f04dd2f46a1014a6b726ad1f63152d3f9a",
    "droplet_kernel<2,3,0>": "afa90341f7545be6898559033dae661be7cc4622f477defa6254e75cb553f532",
    "droplet_kernel<2,3,1>": "10578b9b9d887e02d3a40d348652faa535717ebf92ef2779942930d533f86055",
    "droplet_kernel<4,3,0>": "e813492028544f6899e791a1e8a9fb29dde0f43f1415cae5ea692906159244d7",
    "droplet_kernel<4,3,1>": "a96ff6c9d0ca91c4a5ef059a6e690f1a154957c14e2b6bd0ffb78be2584b36b1",
    "droplet_kernel<8,3,0>": "17a690aedfee3bcb7dfc0e2580a57e1f3dba672ae5f31372aca6ec4724eae3aa",
    "droplet_kernel<8,3,1>": "aa07b96d494d5c9e1f35a7fb3fe5ead89eaadd3ae77143b36f5c66ae1781626d",
    "droplet_kernel<16,3,0>": "c20fcaa93658e9553373223037b113f318e2fef87de548a7bae64165613c3414",
    "droplet_kernel<16,3,1>": "36690f2312362d7be7e0f61613ddfd3a1258f6b2c3a6ab925ff972f348ec86ac",
    "droplet_kernel<32,3,0>": "05a738716ac93d97bd88822310f59e9d654ec7826497b570b0d241a134afbb45",
    "droplet_kernel<32,3,1>": "22736e57d3b457fcb9329ade2376233eb1a2b4388523b6e21dd573a4afceb3d9",
    "droplet_kernel<8,4,0>": "448d6eb5fe984a7b1f8f1a124a2a3b939cc0ce96dc40ae51a0df584bda60ec4f",
    "droplet_kernel<8,4,1>": "580f607b8ad2fef7e6025ec4f648a352098b9f981ee9a3646550f210e3bc4181",
    "droplet_kernel<32,5,0>": "3ff0190715fc2f82aecce59038d89918023a9cdc96f581f2b2ff29334c866fc5",
    "glaciate_mesh_kernel": "8d7e0cac7cdc6811fa15a3ddb8748ecfd79ed13620f9e201636f0a0e9f6ea0ce",
}


def kernel_sass(lib):
    """{short kernel name: SHA-256 of its SASS instruction words} for the droplet and glaciation kernels; the variants the job added carry a ",1" / "<1>"."""
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    res, name, buf = {}, None, []

    def flush():
        if name:
            res[name] = hashlib.sha256("\n".join(buf).encode()).hexdigest()
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            flush()
            f, buf, name = m.group(1), [], None
            t = re.search(r"14droplet_kernelILi(\d+)ELi(\d)ELb(\d)E(?:Lb(\d)E)?E", f)
            g = re.search(r"20glaciate_mesh_kernel(?:ILb(\d)EE)?", f)
            if t:
                name = "droplet_kernel<%s,%s,%s%s>" % (t.group(1), t.group(2), t.group(3), "" if t.group(4) in (None, "0") else "," + t.group(4))
            elif g:
                name = "glaciate_mesh_kernel" + ("" if g.group(1) in (None, "0") else "<1>")
        elif name:
            buf.extend(re.findall(r"/\* (0x[0-9a-f]{16}) \*/", line))   # the instruction words only: cuobjdump also prints section headers that name source paths
    flush()
    return res


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvcc") is None, reason="CUDA toolkit not installed")
def test_existing_kernels_keep_their_sass(tw):
    release = re.search(r"release (\d+\.\d+)", subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout)
    if not release or release.group(1) != SASS_CUDA:
        pytest.skip("the digests are those of CUDA %s" % SASS_CUDA)
    got = kernel_sass(tw.LIB_PATH)
    assert {k: got.get(k) for k in SASS_PARENT} == SASS_PARENT
    assert {k for k in got if k not in SASS_PARENT} == {"droplet_kernel<32,0,1,1>", "droplet_kernel<32,3,0,1>", "droplet_kernel<32,3,1,1>",
                                                        "droplet_kernel<32,5,0,1>", "glaciate_mesh_kernel<1>"}
