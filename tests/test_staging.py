"""CPU checks of csrc/staging.h, the layout every library call gives its buffers: a g++ shim (tests/stagingcheck) runs carves
on null bases, so each take's pointer is its offset.  The CUDA runtime is linked only to resolve symbols; no CUDA call is
reached, so no device is needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA = "/usr/local/cuda"
IN, IO, OUT, DEV = 0, 1, 2, 3
OVS_ERR_UNSUPPORTED = -6
SIZE_T = C.c_size_t


@pytest.fixture(scope="module")
def sc(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("stagingcheck") / "libstagingcheck.so")
    subprocess.check_call(["g++", "-O1", "-fPIC", "-std=c++17", "-shared", "-I" + os.path.join(CUDA, "include"), "-o", so,
                           os.path.join(HERE, "stagingcheck", "stagingcheck.cpp"), "-L" + os.path.join(CUDA, "lib64"), "-lcudart",
                           "-Wl,-rpath," + os.path.join(CUDA, "lib64")])
    lib = C.CDLL(so)
    lib.sc_stage.restype = C.c_int
    lib.sc_error.restype = C.c_char_p
    return lib


def _arrays(takes):
    assert len(takes) <= 64
    kind = np.array([t[0] for t in takes], np.int32)
    elem = np.array([t[1] for t in takes], np.int32)
    count = np.array([t[2] for t in takes], np.uint64)
    return kind, elem, count


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def carve(sc, takes):
    kind, elem, count = _arrays(takes)
    n = len(takes)
    h_off, d_off, h_end = (np.zeros(max(n, 1), np.uint64) for _ in range(3))
    summary = np.zeros(5, np.uint64)
    sc.sc_carve(_ptr(kind), _ptr(elem), _ptr(count), n, _ptr(h_off), _ptr(d_off), _ptr(h_end), _ptr(summary))
    return h_off[:n].astype(np.int64), d_off[:n].astype(np.int64), h_end[:n].astype(np.int64), [int(v) for v in summary]


# (kind, element bytes, count) of some of the library's calls at n elements
def _pose(n):
    return [(IN, 8, 3 * n), (IN, 4, 2 * n), (IN, 4, n), (IN, 4, n), (IO, 8, 12), (IO, 8, 16), (OUT, 1, n), (DEV, 8, 3 * n), (DEV, 1, n)]


def _transform(n):
    return [(IN, 8, 3 * n), (IN, 4, 2 * n), (IN, 4, n)] * 2 + [(IO, 8, 13), (IO, 8, 16), (OUT, 1, n), (DEV, 8, 4 * n), (DEV, 1, n)]


def _stereo(n):
    return [(IN, 1, 32 * n), (IN, 1, 32 * n)] + [(IN, 4, n)] * 6 + [(OUT, 4, n)] * 3 + [(DEV, 4, n)]


def _triangulation(n):
    return [(IN, 1, 32 * n), (IN, 1, 32 * n), (IN, 8, 3 * n), (IN, 8, 3 * n), (IN, 8, n), (IN, 4, n), (IN, 1, n), (IN, 1, n), (OUT, 1, n)]


def _random(seed):
    rng = np.random.default_rng(seed)
    kinds = np.sort(rng.integers(0, 4, int(rng.integers(1, 40))))
    return [(int(k), int(rng.choice([1, 2, 4, 8, 16])), int(rng.choice([0, 1, 3, 255, 256, 257, int(rng.integers(0, 100000))])))
            for k in kinds]


LAYOUTS = ([(f.__name__[1:], n, f(n)) for f in (_pose, _transform, _stereo, _triangulation) for n in (1, 5, 1000, 4097)]
           + [("random", s, _random(s)) for s in range(40)])


@pytest.mark.parametrize("name,n,takes", LAYOUTS, ids=["%s-%d" % (name, n) for name, n, _ in LAYOUTS])
def test_carve_layout(sc, name, n, takes):
    h_off, d_off, h_end, (ordered, up_end, down_begin, h_size, d_size) = carve(sc, takes)
    assert ordered == 1
    kinds = [t[0] for t in takes]
    nbytes = [t[1] * t[2] for t in takes]
    mirrored = [i for i, k in enumerate(kinds) if k != DEV]
    for i in mirrored:
        assert h_off[i] == d_off[i], i                  # one offset on both sides: one copy each way moves them
    for i in range(len(takes)):
        assert d_off[i] % 256 == 0 and (kinds[i] == DEV or h_off[i] % 256 == 0), i
    # no two buffers overlap, on either side
    for side, ids in ((d_off, list(range(len(takes)))), (h_off, mirrored)):
        for a, b in zip(ids, ids[1:]):
            assert side[b] >= side[a] + nbytes[a], (a, b)
    assert d_size == d_off[-1] + nbytes[-1]
    # device takes never move the host arena
    for i, k in enumerate(kinds):
        if k == DEV:
            assert h_end[i] == (h_end[i - 1] if i else 0), i
    assert h_size == (h_end[-1] if takes else 0)
    # upload: everything up to the last in/out byte (the last input byte without one)
    up = [i for i, k in enumerate(kinds) if k in (IN, IO)]
    assert up_end == (h_off[up[-1]] + nbytes[up[-1]] if up else 0)
    # download: from the first in/out buffer (or the first output) to the last output byte (or the last in/out byte)
    down = [i for i, k in enumerate(kinds) if k in (IO, OUT)]
    if down:
        assert down_begin == h_off[down[0]]
        assert h_size == h_off[down[-1]] + nbytes[down[-1]]
        assert all(down_begin <= h_off[i] and h_off[i] + nbytes[i] <= h_size for i in down)
        assert all(h_off[i] + nbytes[i] <= down_begin for i, k in enumerate(kinds) if k == IN)
    assert all(h_off[i] + nbytes[i] <= up_end for i in up)
    assert all(h_off[i] >= up_end for i, k in enumerate(kinds) if k == OUT)


# every take that comes after one of a later kind: in after io / out / dev, io after out / dev, out after dev
OUT_OF_ORDER = [(a, b) for a in (IO, OUT, DEV) for b in (IN, IO, OUT) if b < a]


@pytest.mark.parametrize("first,second", OUT_OF_ORDER)
def test_out_of_order_carve_is_refused_before_any_allocation(sc, first, second):
    for takes in ([(first, 8, 10), (second, 4, 10)],
                  [(IN, 8, 100), (first, 4, 7), (second, 1, 3), (OUT, 8, 2)],
                  _pose(50)[:4] + [(first, 8, 1), (second, 16, 5)] + [(DEV, 8, 20)]):
        assert carve(sc, takes)[3][0] == 0, takes
        kind, elem, count = _arrays(takes)
        allocated = C.c_int(-1)
        assert sc.sc_stage(_ptr(kind), _ptr(elem), _ptr(count), len(takes), C.byref(allocated)) == OVS_ERR_UNSUPPORTED
        assert allocated.value == 0
        assert b"out of order" in sc.sc_error()
