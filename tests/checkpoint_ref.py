"""An independent numpy reading of the checkpoint file format (include/sphk.h, "checkpoints"; DESIGN.md section 2.14): the section
checksum, the header layout and its CRC-32 (zlib's), and a parser that returns the config record and every section's bytes."""
import struct
import zlib

import numpy as np

GAMMA = np.uint64(0x9E3779B97F4A7C15)
MAGIC = b"SPHKCKPT"
VERSION = 1
CONFIG_BYTES = 152
FIXED = 40 + CONFIG_BYTES
ENTRY = 64
CONFIG_FIELDS = [("solver", "16s"), ("capacity_fluid", "i"), ("capacity_boundary", "i"), ("n_boundary", "i"), ("n_bodies", "i"),
                 ("cell_size", "3i"), ("flags", "i"), ("space_size", "3f"), ("cell_length", "f"), ("radius", "f"), ("dt", "f"),
                 ("m0", "f"), ("rho0", "f"), ("rho_boundary", "f"), ("stiff", "f"), ("visc", "f"), ("surface_tension", "f"),
                 ("air_pressure", "f"), ("gravity", "3f"), ("solver_args", "4f"), ("bodies_hash", "Q"), ("open_hash", "Q"),
                 ("settings_hash", "Q")]


def splitmix64(z: np.ndarray) -> np.ndarray:
    z = z.astype(np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def checksum(data) -> int:
    """sum_i splitmix64(w_i + (i + 1) * GAMMA) mod 2^64 over the little-endian u64 words of the zero-padded bytes"""
    b = bytes(data)
    b += b"\0" * (-len(b) % 8)
    w = np.frombuffer(b, "<u8")
    i = np.arange(1, w.size + 1, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return int(splitmix64(w + i * GAMMA).sum(dtype=np.uint64)) if w.size else 0


def crc32(data) -> int:
    return zlib.crc32(bytes(data)) & 0xFFFFFFFF


def header_bytes(n_sections: int) -> int:
    return (FIXED + ENTRY * n_sections + 8 + 15) // 16 * 16


def parse_config(raw: bytes) -> dict:
    out, at = {}, 0
    for name, fmt in CONFIG_FIELDS:
        size = struct.calcsize("<" + fmt)
        v = struct.unpack_from("<" + fmt, raw, at)
        out[name] = v[0].rstrip(b"\0").decode() if fmt == "16s" else (v if len(v) > 1 else v[0])
        at += size
    assert at == CONFIG_BYTES
    return out


def parse(data: bytes, verify: bool = True) -> dict:
    """{"version", "config", "config_raw", "sections": {name: {"offset", "bytes", "elem", "host", "checksum", "data"}}} (in file
    order); verify: raise ValueError on a bad magic, version, CRC, size or checksum"""
    if len(data) < FIXED or data[:8] != MAGIC:
        raise ValueError("bad magic")
    version, n, hb, file_bytes, cfg_hash = struct.unpack_from("<IIQQQ", data, 8)
    if version != VERSION:
        raise ValueError(f"version {version}")
    crc_at = FIXED + ENTRY * n
    (crc,) = struct.unpack_from("<I", data, crc_at)
    if verify and (crc != crc32(data[:crc_at]) or hb != header_bytes(n) or file_bytes != len(data)
                   or cfg_hash != checksum(data[40:FIXED])):
        raise ValueError("header check failed")
    sections = {}
    for k in range(n):
        name, off, size, elem, host, ck = struct.unpack_from("<32sQQIIQ", data, FIXED + ENTRY * k)
        body = data[off:off + size]
        if verify and checksum(body) != ck:
            raise ValueError(f"checksum of {name}")
        sections[name.rstrip(b"\0").decode()] = {"offset": off, "bytes": size, "elem": elem, "host": host, "checksum": ck, "data": body}
    return {"version": version, "config": parse_config(data[40:FIXED]), "config_raw": data[40:FIXED], "sections": sections}


def with_header(data: bytes, **changes) -> bytes:
    """the file with header fields replaced (magic, version) and the CRC recomputed"""
    b = bytearray(data)
    if "magic" in changes:
        b[:8] = changes["magic"]
    if "version" in changes:
        struct.pack_into("<I", b, 8, changes["version"])
    (n,) = struct.unpack_from("<I", b, 12)
    crc_at = FIXED + ENTRY * n
    struct.pack_into("<I", b, crc_at, crc32(b[:crc_at]))
    return bytes(b)


def synthetic(sections, config: bytes = b"\0" * CONFIG_BYTES) -> bytes:
    """a well-formed file of host sections [(name, bytes)] with the given config record (for the device-free refusal tests)"""
    n = len(sections)
    hb = header_bytes(n)
    table, payload, off = b"", b"", hb
    for name, body in sections:
        table += struct.pack("<32sQQIIQ", name.encode(), off, len(body), 1, 1, checksum(body))
        pad = body + b"\0" * (-len(body) % 16)
        payload += pad
        off += len(pad)
    head = MAGIC + struct.pack("<IIQQQ", VERSION, n, hb, hb + len(payload), checksum(config)) + config + table
    head += struct.pack("<I", crc32(head)) + b"\0" * 4
    head += b"\0" * (hb - len(head))
    return head + payload
