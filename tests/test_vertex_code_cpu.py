"""The exact code of k_skin's vertex blocks (fyrox_b200/csrc/fyx_vcode.cuh), run through its host build: every coded block
decodes to the raw block bit for bit, and each block lands on the coded / raw decision the format prescribes."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from fyrox_b200 import _lib
from fyrox_b200.scenegen import Scene
from skin_cases import SkinScene, Surf, unpack_vertices

CSRC = os.path.join(os.path.dirname(_lib.LIB_PATH), "..", "csrc")
VCODE_PATH = os.path.join(os.path.dirname(_lib.LIB_PATH), "libfyrox_vcode.so")

RAW, CODED = 0, 1
RAW_BYTES, CODED_BYTES = 5632, 5136
FLT_MIN, FLT_MAX = 0x00800000, 0x7F7FFFFF


@pytest.fixture(scope="module")
def vc():
    if not os.path.exists(VCODE_PATH):
        subprocess.run(["make", "-C", CSRC, os.path.relpath(VCODE_PATH, CSRC)], check=True, capture_output=True)
    L = C.CDLL(VCODE_PATH)
    L.fyx_vcode_load_surface.restype = C.c_uint32
    L.fyx_vcode_load_surface.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int]
    L.fyx_vcode_decode_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    assert L.fyx_vcode_coded_block_bytes() == CODED_BYTES
    return L


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def codable(raw):
    """numpy statement of the rule, per block of raw (n, 11, 128): every float row's values are +-0 or normal with an exponent
    field within 14 of the row's largest, which is at most 142"""
    v = raw[:, :10]
    e = (v >> 23) & 0xFF
    E = e.max(axis=2, keepdims=True)
    ok = ((v << 1) == 0) | ((e >= 1) & (e + 14 >= E) & (E <= 142))
    return ok.all(axis=(1, 2))


class Blocks:
    """The device's vertex blocks of a sequence of surfaces: each surface padded to 4 vertices and loaded in order
    (k_deinterleave writes its vertices raw, then k_vcode codes the blocks it completes)."""

    def __init__(self, vc, n_verts_total, code=True):
        self.vc = vc
        self.code = code  # False: a context with a palette of more than 64 bones keeps every block raw
        self.n_blocks = (n_verts_total + 127) // 128 + 1
        self.rows = np.zeros((11, self.n_blocks * 128), np.uint32)  # what was loaded, vertex by vertex
        self.dev = np.zeros((self.n_blocks, 11, 128), np.uint32)  # the blocks as the device holds them
        self.flag = np.zeros(self.n_blocks, np.uint8)
        self.spans = []  # (first vertex, end, n_bones) per surface
        self.off = 0

    def add(self, rows, n_bones):
        """rows: (11, n) uint32, the 10 float rows' bits and the bone-index words of the surface's vertices"""
        n = rows.shape[1]
        padded = (n + 3) & ~3
        self.rows[:, self.off:self.off + n] = rows
        v = np.arange(self.off, self.off + padded)
        self.dev[v // 128, :, v % 128] = self.rows[:, v].T
        coded = self.vc.fyx_vcode_load_surface(self.dev.ctypes.data, self.flag.ctypes.data, self.off, padded, int(self.code))
        self.spans.append((self.off, self.off + padded, n_bones))
        self.off += padded
        return coded

    def raw(self):
        return self.rows.reshape(11, self.n_blocks, 128).transpose(1, 0, 2)

    def check(self):
        """bit-exact round trip, and each block's decision against the rule"""
        dec, flag = self.dev.copy(), self.flag.copy()
        self.vc.fyx_vcode_decode_blocks(dec.ctypes.data, flag.ctypes.data, self.n_blocks)
        assert dec.tobytes() == np.ascontiguousarray(self.raw()).tobytes() and (flag == RAW).all()
        fits = codable(self.raw())
        for b in range(self.n_blocks):
            lo, hi = 128 * b, 128 * b + 128
            owners = [s for s, e, _ in self.spans if s < hi and e > lo]
            # untouched, incomplete (it waits for the next surface), outside the code, or a context kept raw
            expect = CODED if owners and hi <= self.off and fits[b] and self.code else RAW
            assert self.flag[b] == expect, (b, owners)

    def coded_bytes(self, b):
        return self.dev[b].tobytes()[:CODED_BYTES]


def rows_of(pos, nrm, w, idx):
    """(n,3), (n,3), (n,4) float32 and (n,) uint32 -> (11, n) uint32"""
    return np.concatenate([bits(pos).T, bits(nrm).T, bits(w).T, np.asarray(idx, np.uint32)[None, :]]).astype(np.uint32)


def plain_rows(n, rng):
    pos = rng.uniform(-4, 4, (n, 3)).astype(np.float32)
    nrm = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    nrm = np.where(np.abs(nrm) < 2.0 ** -10, np.float32(0.5), nrm)  # keep every block codable unless a case says otherwise
    pos = np.where(np.abs(pos) < 2.0 ** -8, np.float32(1.5), pos)
    w = rng.uniform(0.05, 1, (n, 4)).astype(np.float32)
    return rows_of(pos, nrm, w, rng.integers(0, 64, n, dtype=np.uint32) * 0x01010101)


def one_block(vc, rows):
    b = Blocks(vc, 128)
    b.add(rows, 64)
    b.check()
    return b


def set_values(rows, row, vals, start=0):
    r = rows.copy()
    r[row, start:start + len(vals)] = np.asarray(vals, np.uint32)
    return r


def test_plain_block_is_coded_and_exact(vc):
    b = one_block(vc, plain_rows(128, np.random.default_rng(1)))
    assert b.flag[0] == CODED and b.flag[1] == RAW


def test_signed_zeros_in_every_row(vc):
    rows = plain_rows(128, np.random.default_rng(2))
    for r in range(10):
        rows = set_values(rows, r, [0x00000000, 0x80000000], start=2 * r)
    b = one_block(vc, rows)
    assert b.flag[0] == CODED
    rows[:10, :] = np.where(np.arange(128) % 2 == 0, 0x00000000, 0x80000000)  # a block of nothing but +-0
    assert one_block(vc, rows).flag[0] == CODED


@pytest.mark.parametrize("row", [0, 4, 9])
@pytest.mark.parametrize(
    "vals,coded",
    [
        ([0x00000001], False),  # the smallest denormal
        ([0x007FFFFF], False),  # the largest denormal
        ([0x80400000], False),  # a negative denormal
        ([FLT_MIN, FLT_MIN + 7], True),  # exponent field 1 in a row of them
        ([FLT_MAX, FLT_MAX - 1], False),  # beyond 2^16: the scale 2^(E - 15) would not be a float
        ([0x477FFFFF, 0x47000000], True),  # the largest exponent field that codes, 142
        ([0x7F800000], False),  # +Inf
        ([0x7FC00000], False),  # NaN
    ],
)
def test_extreme_values(vc, row, vals, coded):
    base = np.zeros((11, 128), np.uint32)
    base[:10] = bits(np.float32(1.0))
    if vals[0] in (FLT_MIN, FLT_MAX, 0x477FFFFF):  # the whole row at that exponent
        base[row] = vals[0]
    b = one_block(vc, set_values(base, row, vals, start=17))
    assert b.flag[0] == (CODED if coded else RAW)


@pytest.mark.parametrize("row", [1, 5, 8])
def test_exponent_spread_15_fits_16_does_not(vc, row):
    base = plain_rows(128, np.random.default_rng(3))
    base[row] = bits(np.float32(1.0))
    hi = bits(np.float32(1.75))  # exponent field 127
    lo15 = bits(np.float32(2.0 ** -14 * 1.25))  # field 113 = 127 - 14: code 15, the spread of 15 exponents
    lo16 = bits(np.float32(2.0 ** -15 * 1.25))  # field 112: 16 exponents
    b = one_block(vc, set_values(base, row, [hi, lo15, lo15 | 0x80000000], start=40))
    assert b.flag[0] == CODED
    b = one_block(vc, set_values(base, row, [hi, lo16], start=40))
    assert b.flag[0] == RAW


def test_header_and_codes(vc):
    """the pinned layout: E_r in the header after the 10 rows; a group's 40 words in its column; 24-bit values, nibbles"""
    rows = np.zeros((11, 128), np.uint32)
    rows[:10] = bits(np.float32(3.0))  # field 128
    rows[2, 5] = bits(np.float32(-0.75))  # field 126 -> k = 13; vertex 5 = group 1, vertex 1
    rows[10] = np.arange(128, dtype=np.uint32)
    b = one_block(vc, rows)
    assert b.flag[0] == CODED
    blk = b.coded_bytes(0)
    hdr = blk[5120:5136]
    assert list(hdr[:10]) == [128] * 10 and hdr[10:] == b"\0" * 6
    words = np.frombuffer(blk[:5120], np.uint32).reshape(10, 32, 4)
    w = words[:, 1, :].reshape(40)  # group 1
    L1 = ((int(w[6]) >> 24) | (int(w[7]) << 8)) & 0xFFFFFF  # row 2, vertex 1: k & 1 and the mantissa of 0.75
    assert L1 == (1 << 23 | 0x400000)
    nib = (int(w[30 + 1]) >> 8) & 0xF  # rows 2, 3: row 2 in the low nibble of byte 1
    assert nib == (1 << 3 | 13 >> 1)
    assert list(w[35:39]) == [4, 5, 6, 7] and w[39] == 0


def test_shared_blocks_and_padding(vc):
    """blocks that hold the tail of one surface and the head of the next, padding vertices (surfaces of n != 0 mod 4), and the
    last, incomplete block; the same surfaces in a context kept raw"""
    rng = np.random.default_rng(4)
    sizes = [301, 50, 1000, 130, 999, 4, 257, 600, 129]
    surfs = [plain_rows(n, rng) for n in sizes]
    for code in (True, False):
        b = Blocks(vc, sum((n + 3) & ~3 for n in sizes), code)
        for rows in surfs:
            b.add(rows, 64)
        b.check()
        shared = [blk for blk in range(b.n_blocks) if b.flag[blk] == CODED and sum(s < 128 * blk + 128 and e > 128 * blk for s, e, _ in b.spans) > 1]
        assert (len(shared) >= 3) == code


def test_skin_case_surfaces(vc):
    """the vertices of the GPU skinning tests (tests/skin_cases.py: signed zeros, subnormals, extreme positions), every
    palette band and layout, in one context"""
    sc = SkinScene(7, n_bones=300)
    specs = [Surf(nb, n, layout) for nb, n, layout in [(1, 1, "animated"), (63, 127, "k16"), (64, 129, "packed52"), (64, 5000, "animated"),
                                                       (100, 8196, "wide96"), (255, 333, "animated"), (64, 4097, "k16"), (65, 77, "packed52")]]
    specs.append(Surf(64, 3000, "animated", extreme=True))
    b = Blocks(vc, sum((s.n_verts + 3) & ~3 for s in specs))
    for spec in specs:
        sd = sc.make_surface(spec)
        pos, nrm, w, bi = unpack_vertices(sd.verts, spec.layout)
        b.add(rows_of(pos, nrm, w, np.ascontiguousarray(bi).view(np.uint32)[:, 0]), spec.n_bones)
    b.check()
    # the same surfaces without their subnormals: most blocks code
    b2 = Blocks(vc, b.off)
    for s, e, nb in b.spans:
        rows = b.rows[:, s:e].copy()
        sub = ((rows[:10] >> 23) & 0xFF == 0) & ((rows[:10] << 1) != 0)
        rows[:10][sub] = 0
        b2.add(rows, nb)
    b2.check()
    assert (b2.flag == CODED).sum() >= 40


def c4_unit_rows(buf, n):
    rec = buf.reshape(n, 68)  # AnimatedVertex: position, uv, normal, tangent, weights (f32), 4 u8 bone indices
    f = rec[:, :64].copy().view(np.uint32)
    idx = rec[:, 64:68].copy().view(np.uint32)[:, 0]
    return np.concatenate([f[:, 0:3].T, f[:, 5:8].T, f[:, 12:16].T, idx[None, :]]).astype(np.uint32)


def test_c4_scene_round_trip_and_rate(vc):
    """every vertex of the first 2 000 units of the benchmark's default workload (10M nodes, 50k units x 64 bones x 5 000
    vertices, the generator's seed): bit-exact round trip, and the share of raw blocks and the bytes per vertex it comes to"""
    sc = Scene(10_000_000, n_units=50_000, verts_per_unit=5000, bones_per_unit=64)
    V = 5000
    n_coded = n_blocks = 0
    for u0 in range(0, 2000, 32):  # 32 units (or the last 16) are whole blocks: the chunks sit where they do on the device
        per = min(32, 2000 - u0)
        buf = np.empty(per * V * 68, np.uint8)
        sc.units_vertices_into(u0, per, buf.ctypes.data, np.empty(per * 6, np.float32))
        rows = c4_unit_rows(buf, per * V)
        b = Blocks(vc, per * V)
        for u in range(per):
            b.add(rows[:, u * V:(u + 1) * V], 64)
        b.check()
        whole = per * V // 128
        n_coded += int((b.flag[:whole] == CODED).sum())
        n_blocks += whole
    sc.close()
    raw_frac = 1 - n_coded / n_blocks
    bytes_per_vertex = (n_coded * CODED_BYTES + (n_blocks - n_coded) * RAW_BYTES) / (n_blocks * 128)
    print(f"C4, first 2000 units: {n_blocks} blocks, {100 * raw_frac:.2f} % raw, {bytes_per_vertex:.2f} B/vertex read (44 raw)")
    assert raw_frac < 0.10 and bytes_per_vertex < 41.0
