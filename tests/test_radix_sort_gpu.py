"""GPU suite for the project's own radix sort (csrc/radix_sort.cu) through sb_radix_sort_pairs.

The oracle is numpy: with the digit key (k >> begin) & mask, the expected permutation is its stable argsort, and the
expected outputs are the full keys and the payload (or the index) in that order, compared bit for bit.  Covered:
sizes on both sides of every power-of-two sort-tile size from 256 to 16K keys, of the 64K switch between tile sizes
and of 2^20, and one past 2^24 (thousands of tiles, so look-back chains far longer than its window); the key
distributions of the depth sort (float depth bits with culled keys equal to the tile padding), the tile sort (90 % of
the instances in one tile) and the mesh-evaluation grid, plus the distributions where a digit pass goes wrong (equal,
two-valued, sorted, one varying byte, bits outside the sorted range); every bit range of 1 to 32 bits, also starting
past bit 0; a made-up and a given payload; a device-side count from -1 past the capacity; side streams and CUDA-graph
replays.  Every call leaves its inputs byte-identical and writes nothing at or past n."""
import functools
import zlib

import numpy as np
import pytest
import torch

from splatam_b200 import _lib

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5A5A5A5
CULLED = 0xFFFFFFFF           # project.cu's key of a culled Gaussian, and the sort's padding of the last tile
TEMP_FILL = 0xAB              # the temp's content before a call: the sort must zero its own status words

RANGES = [(0, 32), (0, 1), (0, 7), (0, 8), (0, 9), (0, 12), (0, 16), (0, 17), (0, 24), (0, 26), (0, 28), (0, 31),
          (4, 32), (8, 24), (31, 32)]
SIZES = [1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4095, 4096, 4097, 8191, 8192, 8193, 16383, 16384, 16385,
         65535, 65536, 65537, 131071, 131072, 131073, (1 << 20) - 1, (1 << 20) + 1, (1 << 24) + 3]
KINDS = ["random", "equal", "all_culled", "culled_30pct", "zeros", "two_values", "ascending", "descending",
         "byte0", "byte1", "byte2", "byte3", "depth", "tile_90pct", "outside_bits"]
TILES_1200x680, TILES_4112x4112 = 75 * 43, 257 * 257     # 12 and 17 tile-sort bits


def _rng(*key):
    return np.random.default_rng([zlib.crc32(str(k).encode()) for k in key])


@functools.lru_cache(maxsize=None)
def keys_of(kind, n, begin=0, end=32):
    """Keys of one kind, generated once per module (the range matters only to "outside_bits")."""
    rng = _rng("keys", kind, n, begin if kind == "outside_bits" else 0, end if kind == "outside_bits" else 0)
    u32 = lambda size: rng.integers(0, 1 << 32, size, dtype=np.uint32)
    if kind == "random":
        k = u32(n)
    elif kind == "equal":
        k = np.full(n, 0x9E3779B9, np.uint32)
    elif kind == "all_culled":
        k = np.full(n, CULLED, np.uint32)
    elif kind == "culled_30pct":
        k = np.where(rng.random(n) < 0.3, np.uint32(CULLED), u32(n))
    elif kind == "zeros":
        k = np.zeros(n, np.uint32)
    elif kind == "two_values":
        k = u32(2)[rng.integers(0, 2, n)]
    elif kind in ("ascending", "descending"):
        k = np.sort(u32(n))
        k = k if kind == "ascending" else k[::-1].copy()
    elif kind.startswith("byte"):             # only byte b varies: every other pass puts a whole tile in one bin
        b = int(kind[4:])
        k = (np.uint32(0x5A3C96E1) & np.uint32(~(0xFF << (8 * b)) & 0xFFFFFFFF)) | \
            (rng.integers(0, 256, n, dtype=np.uint32) << np.uint32(8 * b))
    elif kind == "depth":                     # the depth sort: float bits of depths in [0.2, 100], a quarter culled
        d = rng.uniform(0.2, 100.0, n).astype(np.float32).view(np.uint32)
        k = np.where(rng.random(n) < 0.25, np.uint32(CULLED), d)
    elif kind == "tile_90pct":                # the tile sort: tile ids of a 4112x4112 view, 90 % in one tile
        k = np.where(rng.random(n) < 0.9, np.uint32(40_000),
                     rng.integers(0, TILES_4112x4112, n, dtype=np.uint32))
    elif kind == "outside_bits":              # digits 0, 1 or all ones, random bits outside [begin, end)
        w = end - begin
        digit = np.array([0, 1, (1 << w) - 1], np.uint64)[rng.integers(0, 3, n)]
        inside = np.uint64(((1 << w) - 1) << begin)
        k = ((u32(n).astype(np.uint64) & ~inside & np.uint64(0xFFFFFFFF)) | (digit << np.uint64(begin)))
        k = k.astype(np.uint32)
    else:
        raise ValueError(kind)
    k.setflags(write=False)
    return k


@functools.lru_cache(maxsize=None)
def payload_of(n):
    v = _rng("payload", n).integers(0, 1 << 32, n, dtype=np.uint32)
    v.setflags(write=False)
    return v


def expected(keys, vals, begin, end, n):
    """numpy's stable argsort of the digit key (k >> begin) & mask over the first n pairs."""
    k = keys[:n]
    digit = (k >> np.uint32(begin)) & np.uint32((1 << (end - begin)) - 1)
    perm = np.argsort(digit, kind="stable")
    return k[perm], (perm.astype(np.uint32) if vals is None else vals[:n][perm])


def _dev(a, dev):
    return torch.from_numpy(np.array(a, dtype=np.uint32).view(np.int32)).to(dev)   # a writable copy


def _host(t):
    return t.cpu().numpy().view(np.uint32)


class Sort:
    """Device buffers of one sort of `capacity` pairs: inputs, sentinel-filled outputs, a temp of exactly the size the
    query gives (filled with junk) and, optionally, the device-side count."""

    def __init__(self, keys, vals, begin, end, dev, capacity=None, n_dev=None):
        self.capacity = len(keys) if capacity is None else capacity
        self.begin, self.end, self.dev = begin, end, dev
        self.kin = _dev(keys, dev)
        self.vin = None if vals is None else _dev(vals, dev)
        m = max(self.capacity, 1)
        self.kout = torch.full((m,), SENTINEL - (1 << 32), dtype=torch.int32, device=dev)
        self.vout = torch.full((m,), SENTINEL - (1 << 32), dtype=torch.int32, device=dev)
        self.temp_bytes = _lib.nbytes("sb_radix_sort_temp_bytes", self.capacity, end - begin)
        self.temp = torch.full((self.temp_bytes,), TEMP_FILL, dtype=torch.uint8, device=dev)
        self.n_dev = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device=dev)

    def reset_outputs(self):
        self.kout.fill_(SENTINEL - (1 << 32))
        self.vout.fill_(SENTINEL - (1 << 32))
        self.temp.fill_(TEMP_FILL)

    def run(self):
        _lib.call("sb_radix_sort_pairs", self.kin, self.vin, self.kout, self.vout, self.capacity, self.n_dev,
                  self.begin, self.end, self.temp, self.temp_bytes, device=self.dev)

    def outputs(self):
        torch.cuda.synchronize(self.dev)
        return _host(self.kout), _host(self.vout)


def check(s, keys, vals, n, what):
    """The first n outputs against the oracle on the first n inputs; the rest of the outputs untouched; the inputs
    byte-identical."""
    ko, vo = s.outputs()
    ek, ev = expected(keys, vals, s.begin, s.end, n)
    assert np.array_equal(ko[:n], ek), "%s: keys differ at %d positions" % (what, int((ko[:n] != ek).sum()))
    assert np.array_equal(vo[:n], ev), "%s: payload differs at %d positions" % (what, int((vo[:n] != ev).sum()))
    assert (ko[n:s.capacity] == SENTINEL).all() and (vo[n:s.capacity] == SENTINEL).all(), "%s: wrote at or past n" % what
    assert np.array_equal(_host(s.kin), keys), "%s: keys_in modified" % what
    if vals is not None:
        assert np.array_equal(_host(s.vin), vals), "%s: vals_in modified" % what


def sort_and_check(keys, vals, begin, end, dev, what):
    s = Sort(keys, vals, begin, end, dev)
    s.run()
    check(s, keys, vals, len(keys), what)


# ---- every size at (0, 32): uniform keys with a given payload, culled keys against the padding and depth keys with
#      the made-up index payload (the depth sort) ------------------------------------------------------------------

@pytest.mark.parametrize("kind,given", [("random", True), ("all_culled", False), ("depth", False)])
@pytest.mark.parametrize("n", SIZES)
def test_every_size_at_32_bits(n, kind, given, cuda_device):
    keys = keys_of(kind, n)
    sort_and_check(keys, payload_of(n) if given else None, 0, 32, cuda_device, "%s n=%d" % (kind, n))


# ---- every key kind and bit range at sizes around tile boundaries, both payloads --------------------------------

BOUNDARY_SIZES = [2047, 4097, 65536, 65537, 131073]


@pytest.mark.parametrize("begin,end", RANGES, ids=["%d-%d" % r for r in RANGES])
@pytest.mark.parametrize("kind", KINDS)
def test_key_kinds_and_bit_ranges(kind, begin, end, cuda_device):
    for n in BOUNDARY_SIZES:
        keys = keys_of(kind, n, begin, end)
        for vals in (None, payload_of(n)):
            sort_and_check(keys, vals, begin, end, cuda_device,
                           "%s n=%d bits [%d,%d) %s payload" % (kind, n, begin, end, "index" if vals is None else "given"))


# ---- the consumers' own calls -----------------------------------------------------------------------------------

def test_depth_sort_call(cuda_device):
    """project.cu: P pairs, 32 bits, the index as payload."""
    P = 1_000_003
    sort_and_check(keys_of("depth", P), None, 0, 32, cuda_device, "depth sort")


@pytest.mark.parametrize("bits,tiles", [(12, TILES_1200x680), (17, TILES_4112x4112)])
def test_tile_sort_call(bits, tiles, cuda_device):
    """binning.cu: R pairs by tile id, the depth-ordered Gaussian ids as payload, the count read on the device (the
    sync-free mode) below, at and past the capacity."""
    R = 2_500_000
    rng = _rng("tile sort", bits)
    keys = np.where(rng.random(R) < 0.3, rng.integers(0, 64, R), rng.integers(0, tiles, R)).astype(np.uint32)
    vals = rng.integers(0, 1_000_000, R, dtype=np.uint32)
    for n in (1_876_543, R, R + 12_345):
        s = Sort(keys, vals, 0, bits, cuda_device, n_dev=n)
        s.run()
        check(s, keys, vals, min(n, R), "tile sort %d bits, n_dev=%d" % (bits, n))


def test_mesh_grid_call(cuda_device):
    """mesh_eval.cu: n cell keys of up to 28 bits, the index as payload."""
    n = 3_000_001
    rng = _rng("grid")
    cells = 400 * 400 * 1600                          # 2.56e8 < 2^28
    keys = np.where(rng.random(n) < 0.5, rng.integers(0, 1000, n), rng.integers(0, cells, n)).astype(np.uint32)
    sort_and_check(keys, None, 0, 28, cuda_device, "mesh grid")


# ---- the device-side count --------------------------------------------------------------------------------------

@pytest.mark.parametrize("capacity", [4097, 65536, 65537, 131073])
@pytest.mark.parametrize("kind,given,begin,end", [("tile_90pct", True, 0, 17), ("depth", False, 0, 32),
                                                  ("random", True, 8, 24)])
def test_device_count(kind, given, begin, end, capacity, cuda_device):
    """*n_dev in {0, 1, tile boundaries, C - 1, C, C + 1, -1, INT_MIN, INT_MAX}: the first clamp(*n_dev, 0, C)
    outputs match the oracle on that many inputs, the rest keep their fill, the inputs stay as they were."""
    keys = keys_of(kind, capacity)
    vals = payload_of(capacity) if given else None
    s = Sort(keys, vals, begin, end, cuda_device, n_dev=0)
    counts = [0, 1, 255, 256, 257, 2047, 2048, 2049, 4095, 4096, 4097, 8192, 16384, 40961, 65535, 65536,
              capacity - 1, capacity, capacity + 1, -1, -(1 << 31), (1 << 31) - 1]
    for c in sorted(set(x for x in counts if x <= capacity + 1 or x == (1 << 31) - 1)):
        s.reset_outputs()
        s.n_dev.fill_(c)
        s.run()
        check(s, keys, vals, min(max(c, 0), capacity), "%s capacity %d, *n_dev=%d" % (kind, capacity, c))


# ---- determinism, streams and CUDA graphs -----------------------------------------------------------------------

def test_repeat_and_side_stream_are_bit_identical(cuda_device):
    n = (1 << 20) + 1
    keys = keys_of("tile_90pct", n)
    s = Sort(keys, None, 0, 17, cuda_device)
    s.run()
    check(s, keys, None, n, "first run")
    first = s.outputs()
    s.reset_outputs()
    s.run()
    again = s.outputs()
    side = torch.cuda.Stream(cuda_device)
    side.wait_stream(torch.cuda.current_stream(cuda_device))
    with torch.cuda.stream(side):
        s.reset_outputs()
        s.run()
    torch.cuda.current_stream(cuda_device).wait_stream(side)
    on_side = s.outputs()
    for got in (again, on_side):
        assert np.array_equal(got[0], first[0]) and np.array_equal(got[1], first[1])


def test_graph_replay_with_new_keys_and_count(cuda_device):
    """One sort captured with a device count; new keys and counts written in place before each replay.  Each replay
    matches the oracle, so the graph re-zeroes the status words and tickets itself."""
    C = 131073
    dev = cuda_device
    keys0 = keys_of("tile_90pct", C)
    vals = payload_of(C)
    s = Sort(keys0, vals, 0, 17, dev, n_dev=100_000)
    s.run()                                           # eager warm-up on the capture device
    check(s, keys0, vals, 100_000, "eager")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        s.run()
    for kind, n in (("random", 70_001), ("depth", C), ("culled_30pct", 4096)):
        keys = keys_of(kind, C)
        s.kin.copy_(_dev(keys, dev))
        s.n_dev.fill_(n)
        s.kout.fill_(SENTINEL - (1 << 32))
        s.vout.fill_(SENTINEL - (1 << 32))
        g.replay()
        check(s, keys, vals, n, "replay with %s keys, n=%d" % (kind, n))


# ---- arguments --------------------------------------------------------------------------------------------------

def test_rejected_calls_and_capacity_zero_write_nothing(cuda_device):
    lib = _lib.load()
    n = 5000
    keys, vals = keys_of("random", n), payload_of(n)
    s = Sort(keys, vals, 0, 32, cuda_device)
    st = _lib.stream(cuda_device)
    p = lambda t: None if t is None else t.data_ptr()
    call = lambda cap, begin, end, temp_bytes, ko=s.kout, vo=s.vout, temp=s.temp: lib.sb_radix_sort_pairs(
        p(s.kin), p(s.vin), p(ko), p(vo), cap, None, begin, end, p(temp), temp_bytes, st)
    assert call(0, 0, 32, 0) == 0
    assert call(n, 0, 32, s.temp_bytes - 1) == 2
    for args in ((n, 0, 0, s.temp_bytes), (n, 0, 33, s.temp_bytes), (n, 16, 8, s.temp_bytes), (1 << 30, 0, 32, 1 << 40)):
        assert call(*args) == 1, args
    assert call(n, 0, 32, s.temp_bytes, temp=None) == 1
    assert call(n, 0, 32, s.temp_bytes, ko=s.kin) == 1
    assert call(n, 0, 32, s.temp_bytes, vo=s.vin) == 1
    check(s, keys, vals, 0, "rejected calls")
    assert (s.temp.cpu() == TEMP_FILL).all()
