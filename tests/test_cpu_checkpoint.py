"""Checkpoints without a device: the library's host checksum and CRC-32 against the numpy restatement (checkpoint_ref.py), and
every refusal of sphk_state_open that needs no device (magic, version, truncated header or payload, header CRC)."""
import ctypes as C

import numpy as np
import pytest

import checkpoint_ref as CR

INVALID = -1


@pytest.fixture(scope="module")
def lib(built):
    from cpp_fluid_particles_b200 import capi
    L = capi.sphk()
    L.sphk_state_checksum_host.argtypes = [C.c_void_p, C.c_ulonglong, C.POINTER(C.c_ulonglong)]
    L.sphk_state_crc32_host.argtypes = [C.c_void_p, C.c_ulonglong, C.POINTER(C.c_uint)]
    L.sphk_state_close.restype = None
    return L


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 15, 16, 17, 4095, 4096, 100003])
def test_host_checksum_and_crc_match_the_reference(lib, n):
    data = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes()
    buf = C.create_string_buffer(data, max(n, 1))
    h, crc = C.c_ulonglong(0), C.c_uint(0)
    assert lib.sphk_state_checksum_host(buf, n, C.byref(h)) == 0 and lib.sphk_state_crc32_host(buf, n, C.byref(crc)) == 0
    assert h.value == CR.checksum(data) and crc.value == CR.crc32(data)


def test_checksum_depends_on_word_position_and_padding(lib):
    a = bytes(range(16))
    assert CR.checksum(a) != CR.checksum(a[8:] + a[:8])          # the word index is mixed in
    assert CR.checksum(b"\1") == CR.checksum(b"\1" + b"\0" * 7)    # a partial word is zero-padded
    assert CR.checksum(b"") == 0


def _open(lib, path):
    f, msg = C.c_void_p(), C.create_string_buffer(512)
    rc = lib.sphk_state_open(str(path).encode(), C.byref(f), msg, C.c_int(512))
    if rc == 0:
        lib.sphk_state_close(f)
    return rc, msg.value.decode()


def test_a_well_formed_file_opens_and_names_its_sections(lib, tmp_path):
    data = CR.synthetic([("system.record", b"\1" * 80), ("user", b"frame 7")])
    p = tmp_path / "ok.ckpt"
    p.write_bytes(data)
    assert _open(lib, p) == (0, "")
    parsed = CR.parse(data)
    assert list(parsed["sections"]) == ["system.record", "user"] and parsed["sections"]["user"]["data"] == b"frame 7"
    f = C.c_void_p()
    assert lib.sphk_state_open(str(p).encode(), C.byref(f), None, C.c_int(0)) == 0
    nb = C.c_ulonglong(0)
    assert lib.sphk_state_section_bytes(f, b"user", C.byref(nb)) == 0 and nb.value == 7
    assert lib.sphk_state_section_bytes(f, b"fluid.pos", C.byref(nb)) == INVALID
    lib.sphk_state_close(f)


@pytest.mark.parametrize("case, words", [
    ("magic", "bad magic"), ("version", "version"), ("truncated_header", "truncated"), ("crc", "CRC"),
    ("truncated_payload", "truncated"), ("missing", "cannot open")])
def test_device_free_refusals(lib, tmp_path, case, words):
    data = CR.synthetic([("system.record", b"\2" * 80), ("user", b"x" * 33)])
    if case == "magic":
        data = CR.with_header(data, magic=b"SPHKCKPX")
    elif case == "version":
        data = CR.with_header(data, version=2)
    elif case == "truncated_header":
        data = data[:100]
    elif case == "crc":
        b = bytearray(data)
        b[CR.FIXED + 40] ^= 1                 # a bit of the first section's offset
        data = bytes(b)
    elif case == "truncated_payload":
        data = data[:-5]
    p = tmp_path / "bad.ckpt"
    if case != "missing":
        p.write_bytes(data)
    rc, msg = _open(lib, p)
    assert rc == INVALID and words in msg, msg


def test_header_fields_are_where_the_reference_reads_them():
    cfg = bytearray(CR.CONFIG_BYTES)
    cfg[:5] = b"dfsph"
    data = CR.synthetic([("user", b"")], bytes(cfg))
    parsed = CR.parse(data)
    assert parsed["config"]["solver"] == "dfsph" and parsed["sections"]["user"]["bytes"] == 0
    assert len(data) == CR.header_bytes(1) and CR.header_bytes(1) % 16 == 0


@pytest.mark.parametrize("extra", [
    ["--checkpoint-every", "5"], ["--checkpoint", "x.ckpt", "--checkpoint-every", "-1"],
    ["--checkpoint", "x.ckpt", "--checkpoint-every", "abc"], ["--checkpoint", "x.ckpt", "--ranks", "2"],
    ["--resume", "x.ckpt", "--ranks", "2"], ["--resume", "x.ckpt", "--bullets", "3"], ["--checkpoint"], ["--resume"]])
def test_headless_refuses_bad_checkpoint_arguments(built, extra):
    """refused while parsing, before any CUDA call"""
    import os
    import subprocess
    from util import ROOT
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    r = subprocess.run([cli, "--frames", "0"] + extra, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 2, r.stderr
