"""CPU suite for the radix sort's checked entry point (sb_radix_sort_temp_bytes, sb_radix_sort_pairs): every argument
is checked before the first CUDA call, and the temp size never decreases as the capacity grows.  The sort itself is
tested against numpy in test_radix_sort_gpu.py."""
import ctypes

from splatam_b200 import _lib

BAD_ARG, WORKSPACE = 1, 2


def _temp_bytes(capacity, bits):
    n = ctypes.c_size_t(0)
    assert _lib.load().sb_radix_sort_temp_bytes(capacity, bits, ctypes.byref(n)) == 0, (capacity, bits)
    return n.value


def test_temp_bytes_never_decrease_as_the_capacity_grows():
    """A temp sized for one capacity must serve every smaller one, also across the switch from 2048-key to 4096-key
    sort tiles at 64K pairs, where the number of look-back status words halves."""
    caps = list(range(0, 140_000)) + [int(c) for c in (1.05 ** k for k in range(245, 425))] + [(1 << 30) - 1]
    caps = sorted(set(c for c in caps if c < 1 << 30))
    for bits in (8, 16, 24, 32):                    # 1 to 4 passes
        prev = 0
        for c in caps:
            b = _temp_bytes(c, bits)
            assert b >= prev, "bits %d: capacity %d needs %d bytes, less than the %d of a smaller one" % (bits, c, b, prev)
            prev = b
        assert prev >= 8 * ((1 << 30) - 1)          # the ping-pong pair buffer at the largest capacity
    for c in (1, 65536, 65537, 1 << 20):            # more passes never need less
        sizes = [_temp_bytes(c, bits) for bits in range(1, 33)]
        assert sizes == sorted(sizes), c


def test_entry_points_check_arguments_before_any_launch():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    for capacity, bits in ((-1, 8), (1 << 30, 8), (16, 0), (16, 33), (16, -1)):
        assert lib.sb_radix_sort_temp_bytes(capacity, bits, ctypes.byref(n)) == BAD_ARG, (capacity, bits)
    assert lib.sb_radix_sort_temp_bytes(16, 8, None) == BAD_ARG
    assert lib.sb_radix_sort_temp_bytes(0, 32, ctypes.byref(n)) == 0

    # Distinct non-null dummy pointers, never dereferenced: every call below returns before any CUDA call.
    K, V, KO, VO, T = 0x1000, 0x2000, 0x3000, 0x4000, 0x5000
    C = 5000
    need = _temp_bytes(C, 32)
    sort = lambda *a: lib.sb_radix_sort_pairs(*a, None)
    # bit range and capacity
    for begin, end in ((0, 0), (0, 33), (8, 8), (9, 8), (-1, 8), (32, 32), (31, 40)):
        assert sort(K, V, KO, VO, C, None, begin, end, T, need) == BAD_ARG, (begin, end)
        assert sort(K, V, KO, VO, 0, None, begin, end, T, need) == BAD_ARG, (begin, end)   # even for no pairs
    assert sort(K, V, KO, VO, -1, None, 0, 32, T, need) == BAD_ARG
    assert sort(K, V, KO, VO, 1 << 30, None, 0, 32, T, 1 << 62) == BAD_ARG
    # capacity 0: nothing to sort, nothing launched, whatever the buffers
    assert sort(None, None, None, None, 0, None, 0, 32, None, 0) == 0
    # null buffers; NULL vals_in (index payload) and NULL n_dev (host count) are allowed
    assert sort(None, V, KO, VO, C, None, 0, 32, T, need) == BAD_ARG
    assert sort(K, V, None, VO, C, None, 0, 32, T, need) == BAD_ARG
    assert sort(K, V, KO, None, C, None, 0, 32, T, need) == BAD_ARG
    assert sort(K, None, KO, VO, C, None, 0, 32, None, need) == BAD_ARG
    # aliasing: an odd pass count writes the outputs in the pass that reads the inputs
    for ko, vo in ((K, VO), (KO, V), (V, VO), (KO, K), (KO, KO)):
        assert sort(K, V, ko, vo, C, None, 0, 32, T, need) == BAD_ARG, (ko, vo)
    # the workspace: one byte short of the size query
    for begin, end in ((0, 32), (0, 8), (4, 32), (8, 24), (31, 32)):
        short = _temp_bytes(C, end - begin) - 1
        assert sort(K, None, KO, VO, C, None, begin, end, T, short) == WORKSPACE, (begin, end)
    assert sort(K, None, KO, VO, 1 << 20, None, 0, 17, T, _temp_bytes(1 << 20, 17) - 1) == WORKSPACE
