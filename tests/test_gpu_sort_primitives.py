"""The library's shared sort, run and scan primitives (csrc/binning.cu), each on its own against exact numpy integer arithmetic,
through the test entry points gof_probe_* (not part of the public header):

- gof_sort_words_u32: stable LSD sort by a key of 1-3 u32 words, only the low bits[k] bits of word k count.  Stable, so the
  order is unique: it must equal np.lexsort of the masked words bit for bit, over odd and even total pass counts (the odd
  count starts the values in the buffer that is not `ord`), ord = va and vb, w[0] == ka (the sort overwrites it) and not,
  garbage above `bits`, ragged tails, chunks with empty digits and heavy duplicates.  It writes no key word except an
  aliased w[0], no byte past any buffer or past gof_sort_scratch_bytes(n) of scratch, and gives the same result whatever
  the buffers held before.
- gof_key_runs_u32: head flags, run numbers (the exclusive scan of the heads) and the run count along an order, comparing
  masked words.
- gof_exclusive_scan_u32: the single-launch decoupled look-back scan, at sizes around its 2048-value chunk and over
  thousands of chunks, and with running totals past 2^30 and up to 2^32 - 1 (exact), reduced mod 2^32 beyond.

The last test needs no device: with no GPU visible, every argument the sort refuses (word count, bit widths, n >= 2^30)
must come back as GOF_E_INVALID, and n = 2^30 - 1 must get past the checks to the first CUDA call."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "gaussian-opacity-fields_b200", "diff_gaussian_rasterization", "libgof_b200.so")
GOF_OK, GOF_E_INVALID, GOF_E_CUDA = 0, -1, -2
SORT_SCRATCH, SCAN_SCRATCH = 0, 1
GUARD = 4096           # bytes of random guard band after every buffer
FILLS = (0x00, 0xFF)   # every call runs twice, over scratch and output buffers pre-filled with each byte

_v = ctypes.c_void_p
_words_t = ctypes.POINTER(ctypes.c_void_p)
_bits_t = ctypes.POINTER(ctypes.c_int)


def _bind(lib):
    lib.gof_probe_sort_words_u32.restype = ctypes.c_int
    lib.gof_probe_sort_words_u32.argtypes = [ctypes.c_int, _words_t, _bits_t, ctypes.c_size_t, _v, _v, _v, _v, _v, ctypes.c_int, _v]
    lib.gof_probe_key_runs_u32.restype = ctypes.c_int
    lib.gof_probe_key_runs_u32.argtypes = [ctypes.c_int, _words_t, _bits_t, _v, ctypes.c_size_t, _v, _v, _v, _v, _v]
    lib.gof_probe_exclusive_scan_u32.restype = ctypes.c_int
    lib.gof_probe_exclusive_scan_u32.argtypes = [_v, _v, _v, _v, ctypes.c_size_t, _v]
    lib.gof_probe_scratch_bytes.restype = ctypes.c_size_t
    lib.gof_probe_scratch_bytes.argtypes = [ctypes.c_int, ctypes.c_size_t]
    lib.gof_last_error.restype = ctypes.c_char_p
    return lib


def _lib():
    from diff_gaussian_rasterization import _C
    return _bind(_C._lib), _C._stream()


class _Buf:
    """A device buffer of `nbytes` bytes followed by GUARD bytes of a seeded random pattern."""

    def __init__(self, nbytes, fill=0, data=None, seed=0):
        self.nbytes = int(nbytes)
        self.guard = torch.randint(0, 256, (GUARD,), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))
        host = torch.empty(self.nbytes + GUARD, dtype=torch.uint8)
        host[:self.nbytes] = fill
        if data is not None:
            host[:self.nbytes] = torch.from_numpy(np.ascontiguousarray(data, dtype=np.uint32).view(np.uint8))
        host[self.nbytes:] = self.guard
        self.t = host.cuda()

    @classmethod
    def u32(cls, data, seed):
        return cls(4 * data.size, data=data, seed=seed)

    def ptr(self):
        return self.t.data_ptr()

    def values(self, count=None):
        count = self.nbytes // 4 if count is None else count
        return self.t[:4 * count].cpu().numpy().view(np.uint32)

    def assert_guard(self, name):
        assert torch.equal(self.t[self.nbytes:].cpu(), self.guard), f"{name}: bytes written past its end"


def _mask(bits):
    return np.uint32((1 << bits) - 1)


def _words_arg(ptrs, bits):
    return (ctypes.c_void_p * 4)(*(list(ptrs) + [None] * (4 - len(ptrs)))), (ctypes.c_int * 4)(*(list(bits) + [0] * (4 - len(bits))))


def _lexsort(words, bits):
    """Stable order by the masked words, w[0] least significant (np.lexsort's LAST key is its primary one)."""
    n = words[0].size
    return np.lexsort([np.arange(n)] + [w & _mask(b) for w, b in zip(words, bits)]).astype(np.uint32)


# ------------------------------------------------------------------------------------------------------------------------
# sort

def _sort_once(lib, stream, words, bits, ord_is_vb, alias, fill):
    n = words[0].size
    b = {name: _Buf(4 * n, fill, seed=i) for i, name in enumerate(("ka", "kb", "va", "vb"))}
    b["hist"] = _Buf(lib.gof_probe_scratch_bytes(SORT_SCRATCH, n), fill, seed=4)
    if alias:
        b["ka"] = _Buf.u32(words[0], seed=0)
    wb = [b["ka"] if (k == 0 and alias) else _Buf.u32(w, seed=10 + k) for k, w in enumerate(words)]
    wp, bp = _words_arg([x.ptr() for x in wb], bits)
    rc = lib.gof_probe_sort_words_u32(len(words), wp, bp, n, b["ka"].ptr(), b["kb"].ptr(), b["va"].ptr(), b["vb"].ptr(),
                                      b["hist"].ptr(), int(ord_is_vb), stream)
    torch.cuda.synchronize()
    assert rc == GOF_OK, lib.gof_last_error()
    for name, x in b.items():
        x.assert_guard(name)
    for k, (w, x) in enumerate(zip(words, wb)):
        if not (k == 0 and alias):
            x.assert_guard(f"w[{k}]")
            np.testing.assert_array_equal(x.values(), w, err_msg=f"the sort wrote key word {k}")
    return b["vb" if ord_is_vb else "va"].values()


def _check_sort(words, bits, ord_is_vb, alias, fills=FILLS):
    lib, stream = _lib()
    want = _lexsort(words, bits)
    for fill in fills:
        got = _sort_once(lib, stream, words, bits, ord_is_vb, alias, fill)
        if not np.array_equal(got, want):
            bad = np.flatnonzero(got != want)
            pytest.fail(f"fill {fill:#x}: {bad.size} of {want.size} positions differ from np.lexsort, first at {bad[0]}: "
                        f"got item {got[bad[0]]}, want {want[bad[0]]}")


def _uniform(rng, n):
    return rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)


def _passes(bits):
    return sum((b + 7) // 8 for b in bits)


# word configurations: per word count one odd and one even total of radix passes, and the three callers' configurations
CONFIGS = [
    (24,),            # 3 passes
    (32,),            # 4
    (5, 32),          # 5
    (32, 31),         # 8: TSDF touch (block key, low and high word)
    (20, 20),         # 6: tetmesh, 2 x bits_for(num_verts)
    (13, 13),         # 4: tetmesh, a smaller mesh
    (8, 8, 8),        # 3
    (9, 1, 13),       # 5
    (7, 31, 1),       # 6
    (32, 32, 32),     # 12: kNN (96-bit Morton key; w[0] is ka)
]
assert {(len(c), _passes(c) % 2) for c in CONFIGS} == {(nw, par) for nw in (1, 2, 3) for par in (0, 1)}


@pytest.mark.gpu
@pytest.mark.parametrize("alias", [False, True], ids=["w0_own", "w0_is_ka"])
@pytest.mark.parametrize("ord_is_vb", [False, True], ids=["ord_va", "ord_vb"])
@pytest.mark.parametrize("bits", CONFIGS, ids=["_".join(map(str, c)) for c in CONFIGS])
def test_sort_word_configs_and_buffers(bits, ord_is_vb, alias):
    """Every word configuration with ord = va / vb and w[0] == ka or not: three chunks and one key, every word uniform over
    all 32 bits (garbage above `bits`)."""
    rng = np.random.default_rng(_passes(bits) * 4 + 2 * ord_is_vb + alias)
    n = 12_289
    _check_sort([_uniform(rng, n) for _ in bits], bits, ord_is_vb, alias)


SIZES = [0, 1, 2, 31, 255, 256, 4095, 4096, 4097, 12_289, 1_000_003]


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_sort_sizes(n):
    """Empty, single-item, single-chunk, exactly-whole-chunk and ragged sizes; odd and even pass counts over 1-3 words, each
    buffer arrangement once."""
    rng = np.random.default_rng(n)
    for bits, ord_is_vb, alias in (((24,), True, True), ((32, 31), False, False), ((9, 1, 13), True, False),
                                   ((32, 32, 32), False, True)):
        _check_sort([_uniform(rng, n) for _ in bits], bits, ord_is_vb, alias)


def _split(bits):
    """Digit widths of the radix passes over one word, low digit first, as evenly as possible (13 -> 7 + 6)."""
    passes, rem, out = (bits + 7) // 8, bits, []
    for p in range(passes):
        w = (rem + (passes - p) - 1) // (passes - p)
        out.append(w)
        rem -= w
    return out


def _distribution(kind, rng, n, bits):
    """n words whose low `bits` bits follow `kind`; random garbage above them."""
    m = int(_mask(bits))
    if kind == "uniform":
        return _uniform(rng, n)
    if kind == "equal":
        low = np.full(n, rng.integers(0, m + 1), dtype=np.uint64)
    elif kind == "two":
        low = rng.choice(rng.integers(0, m + 1, 2, dtype=np.uint64), n)
    elif kind in ("sorted", "reversed"):
        low = np.sort(rng.integers(0, m + 1, n, dtype=np.uint64))
        if kind == "reversed":
            low = low[::-1]
    elif kind == "top":   # only the most significant radix digit varies: every other pass sees one digit, most are empty
        top = _split(bits)[-1]
        low = rng.integers(0, 1 << top, n, dtype=np.uint64) << np.uint64(bits - top)
    elif kind == "small":
        low = rng.integers(0, 16, n, dtype=np.uint64) & np.uint64(m)
    else:
        raise ValueError(kind)
    return ((low & np.uint64(m)) | (_uniform(rng, n).astype(np.uint64) & np.uint64(~m & 0xFFFFFFFF))).astype(np.uint32)


DISTS = ["uniform", "equal", "two", "sorted", "reversed", "top", "small"]
WIDTHS = [1, 7, 8, 9, 13, 31, 32]


@pytest.mark.gpu
@pytest.mark.parametrize("nw", [1, 2])
@pytest.mark.parametrize("bits", WIDTHS)
@pytest.mark.parametrize("dist", DISTS)
def test_sort_key_distributions(dist, bits, nw):
    """Bit widths from 1 to 32 (1 and 2 passes per word, even and uneven digit splits) under distributions that stress the
    ranking and the look-back: all equal, two values, presorted, reversed, only the top digit varying, heavy duplicates."""
    rng = np.random.default_rng(1000 * DISTS.index(dist) + 10 * bits + nw)
    n = 40_961   # ten chunks and one key
    ws = [_distribution(dist, rng, n, bits) for _ in range(nw)]
    case = DISTS.index(dist) + WIDTHS.index(bits)
    _check_sort(ws, (bits,) * nw, ord_is_vb=bool(case & 1), alias=bool(case & 2))


@pytest.mark.gpu
def test_sort_three_words_large():
    """The kNN configuration (3 x 32 bits, 12 passes, w[0] is ka) over 2^24 + 3 items, with duplicates in the top word."""
    rng = np.random.default_rng(24)
    n = (1 << 24) + 3
    ws = [_uniform(rng, n), _uniform(rng, n), rng.integers(0, 1 << 12, n, dtype=np.uint64).astype(np.uint32)]
    _check_sort(ws, (32, 32, 32), ord_is_vb=False, alias=True)


# ------------------------------------------------------------------------------------------------------------------------
# runs of equal keys

def _runs_case(kind):
    rng = np.random.default_rng(len(kind))
    if kind == "empty":
        return [np.zeros(0, np.uint32)], (32,)
    if kind == "one":
        return [_uniform(rng, 1)], (17,)
    if kind == "above_bits":   # keys that differ only above `bits`: one run
        n = 4097
        return [(_uniform(rng, n) << np.uint32(8)) | np.uint32(0x5A), _uniform(rng, n) | np.uint32(0x3FF)], (8, 10)
    if kind == "equal":
        n = 12_289
        return [np.full(n, v, np.uint32) for v in (7, 0xFFFFFFFF, 123456)], (32, 32, 32)
    if kind == "distinct":
        n = 1_000_003
        p = rng.permutation(n).astype(np.uint32)
        return [p & np.uint32(0x3FF), (p >> np.uint32(10)) | (_uniform(rng, n) << np.uint32(10))], (10, 10)
    if kind == "dups":         # many equal keys; some runs break only in the second or third word
        n = 1_000_003
        return [_distribution("small", rng, n, 4), _distribution("small", rng, n, 9), _distribution("two", rng, n, 31)], (4, 9, 31)
    raise ValueError(kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["empty", "one", "above_bits", "equal", "distinct", "dups"])
def test_key_runs(kind):
    lib, stream = _lib()
    words, bits = _runs_case(kind)
    n = words[0].size
    order = _lexsort(words, bits)
    masked = np.stack([w[order] & _mask(b) for w, b in zip(words, bits)])
    head = np.ones(n, np.uint32)
    head[1:] = np.any(masked[:, 1:] != masked[:, :-1], axis=0)
    run = (np.cumsum(head, dtype=np.uint64) - head).astype(np.uint32)
    want_runs = {"empty": 0, "one": 1, "above_bits": 1, "equal": 1, "distinct": n}.get(kind, int(head.sum()))
    assert int(head.sum()) == want_runs
    for fill in FILLS:
        wb = [_Buf.u32(w, seed=10 + k) for k, w in enumerate(words)]
        ob = _Buf.u32(order, seed=20)
        b = dict(head=_Buf(4 * n, fill, seed=1), run=_Buf(4 * n, fill, seed=2),
                 scan_tmp=_Buf(lib.gof_probe_scratch_bytes(SCAN_SCRATCH, n), fill, seed=3), num_runs=_Buf(4, fill, seed=4))
        wp, bp = _words_arg([x.ptr() for x in wb], bits)
        rc = lib.gof_probe_key_runs_u32(len(words), wp, bp, ob.ptr(), n, b["head"].ptr(), b["run"].ptr(), b["scan_tmp"].ptr(),
                                        b["num_runs"].ptr(), stream)
        torch.cuda.synchronize()
        assert rc == GOF_OK, lib.gof_last_error()
        for name, x in b.items():
            x.assert_guard(name)
        np.testing.assert_array_equal(b["head"].values(), head)
        np.testing.assert_array_equal(b["run"].values(), run)
        assert int(b["num_runs"].values()[0]) == want_runs
        for k, (w, x) in enumerate(zip(words, wb)):
            np.testing.assert_array_equal(x.values(), w, err_msg=f"key word {k} written")
        np.testing.assert_array_equal(ob.values(), order, err_msg="ord written")


# ------------------------------------------------------------------------------------------------------------------------
# exclusive scan

def _check_scan(values, fills=FILLS):
    lib, stream = _lib()
    values = np.ascontiguousarray(values, dtype=np.uint32)
    n = values.size
    incl = np.cumsum(values, dtype=np.uint64)
    want = ((incl - values) & 0xFFFFFFFF).astype(np.uint32)
    want_total = int(incl[-1]) & 0xFFFFFFFF if n else 0
    for fill in fills:
        b = dict(inp=_Buf.u32(values, seed=1), out=_Buf(4 * n, fill, seed=2),
                 tmp=_Buf(lib.gof_probe_scratch_bytes(SCAN_SCRATCH, n), fill, seed=3), total=_Buf(4, fill, seed=4))
        rc = lib.gof_probe_exclusive_scan_u32(b["inp"].ptr(), b["out"].ptr(), b["tmp"].ptr(), b["total"].ptr(), n, stream)
        torch.cuda.synchronize()
        assert rc == GOF_OK, lib.gof_last_error()
        for name, x in b.items():
            x.assert_guard(name)
        np.testing.assert_array_equal(b["inp"].values(), values, err_msg="input written")
        got = b["out"].values()
        if not np.array_equal(got, want):
            bad = np.flatnonzero(got != want)
            pytest.fail(f"fill {fill:#x}: {bad.size} of {n} offsets wrong, first at {bad[0]} (chunk {bad[0] // 2048}): "
                        f"got {got[bad[0]]}, want {want[bad[0]]}")
        assert int(b["total"].values()[0]) == want_total, f"fill {fill:#x}: total"


SCAN_SIZES = [0, 1, 2047, 2048, 2049, 4097, 2048 * 257 + 5, 10_000_019]
SCAN_VALUES = {"flags": 2, "counts6": 7, "counts1536": 1537}


@pytest.mark.gpu
@pytest.mark.parametrize("values", list(SCAN_VALUES))
@pytest.mark.parametrize("n", SCAN_SIZES)
def test_exclusive_scan(n, values):
    """Sizes around one 2048-value chunk and over thousands of chunks: 0/1 flags, small counts (marching-tetrahedra
    crossings) and counts up to 1536 (vertices and faces of a TSDF block)."""
    rng = np.random.default_rng(n * 7 + SCAN_VALUES[values])
    _check_scan(rng.integers(0, SCAN_VALUES[values], n).astype(np.uint32))


def _summing_to(total, n, seed):
    return np.random.default_rng(seed).multinomial(total, np.full(n, 1.0 / n)).astype(np.uint32)


def _big_case(kind):
    rng = np.random.default_rng(5)
    if kind == "chunk0_exactly_2pow30":   # 4097 values of 2^19: chunk 0's inclusive prefix is exactly 2^30
        return np.full(4097, 1 << 19, np.uint32)
    if kind == "total_2pow30m1":
        return _summing_to((1 << 30) - 1, 100_003, 1)
    if kind == "total_2pow30":
        return _summing_to(1 << 30, 100_003, 2)
    if kind == "total_2pow31p7":
        return _summing_to((1 << 31) + 7, 2048 * 257 + 5, 3)
    if kind == "total_2pow32m1":   # the largest total a u32 holds
        return _summing_to((1 << 32) - 1, 1_000_003, 4)
    if kind == "big_first":
        v = rng.integers(0, 7, 50_001).astype(np.uint32)
        v[0] = (1 << 30) - 1
        return v
    if kind == "big_last":
        v = rng.integers(0, 7, 50_001).astype(np.uint32)
        v[-1] = (1 << 30) - 1
        return v
    if kind == "wraps_2pow32":     # beyond 2^32 the offsets and the total are reduced mod 2^32, like any u32 sum
        return _summing_to((1 << 32) + 12_345, 300_007, 6)
    raise ValueError(kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["chunk0_exactly_2pow30", "total_2pow30m1", "total_2pow30", "total_2pow31p7", "total_2pow32m1",
                                  "big_first", "big_last", "wraps_2pow32"])
def test_exclusive_scan_totals_past_2pow30(kind):
    """Running totals at and past 2^30 must survive the look-back between chunks: every offset and the total exact below
    2^32 (a 30-bit field in the status word would carry 2^30 into its flag bits and lose it)."""
    _check_scan(_big_case(kind))


# ------------------------------------------------------------------------------------------------------------------------
# limits (no device)

_LIMITS_SCRIPT = textwrap.dedent("""
    import ctypes, json, sys
    sys.path.insert(0, sys.argv[2])
    from test_gpu_sort_primitives import _bind, _words_arg
    lib = _bind(ctypes.CDLL(sys.argv[1]))
    out = {}
    def call(name, nw, bits, n):
        wp, bp = _words_arg([None] * min(nw, 4), bits)
        out[name] = [lib.gof_probe_sort_words_u32(nw, wp, bp, n, None, None, None, None, None, 0, None),
                     lib.gof_last_error().decode()]
    call("nw0", 0, [], 1)
    call("nw4", 4, [8, 8, 8, 8], 1)
    call("bits0", 1, [0], 1)
    call("bits33", 1, [33], 1)
    call("bits0_w2", 3, [8, 8, 0], 1)
    call("bits33_w1", 2, [32, 33], 1)
    call("n_2pow30", 2, [32, 31], 1 << 30)
    call("n_2pow30_nw1", 1, [8], (1 << 30) + 12345)
    call("n_2pow30m1", 2, [32, 31], (1 << 30) - 1)
    print(json.dumps(out))
""")


def test_sort_limits_without_a_device():
    """Runs on the CPU: arguments the sort refuses are refused before any CUDA call, and an n just under the limit gets past
    the checks (and then fails at its first launch: no device is visible)."""
    assert os.path.exists(LIB_PATH), "build the library first: python gaussian-opacity-fields_b200/build.py"
    import json
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _LIMITS_SCRIPT, LIB_PATH, os.path.dirname(os.path.abspath(__file__))],
                         env=env, capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stderr
    out = json.loads(res.stdout.strip().splitlines()[-1])
    for name in ("nw0", "nw4", "bits0", "bits33", "bits0_w2", "bits33_w1", "n_2pow30", "n_2pow30_nw1"):
        assert out[name][0] == GOF_E_INVALID, (name, out[name])
    for name in ("n_2pow30", "n_2pow30_nw1"):
        assert "2^30" in out[name][1], (name, out[name])
    assert out["n_2pow30m1"][0] == GOF_E_CUDA, out["n_2pow30m1"]
