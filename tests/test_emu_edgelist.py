"""The corpus builder's parse (csrc/edgelist.cu) under the CPU emulator, driven chunk by chunk through the product's
ChunkReader with staging chunks of a few hundred bytes, so that lines straddle chunk boundaries and boundaries land
exactly on '\\n'.  The keys, line counts, header values and the first error must equal the Python restatement
(x2dgl_oracle.parse_keys); from_keys_device on CPU tensors must equal synthetic.from_pairs and the reference's own
x2dgl run (tests/golden/x2dgl_golden.npz)."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

import x2dgl_oracle as oracle
from emu_util import lib, ptr
from gcc_b200 import _capi
from gcc_b200.datasets import synthetic
from gcc_b200.datasets.x2dgl import ChunkReader, LineTooLong

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "x2dgl_golden.npz")
NONE = (1 << 64) - 1


def emu_parse(data, fmt, chunk):
    L = lib()
    ws_bytes = L.gccb_edgelist_workspace(chunk)
    ws = np.zeros(ws_bytes, np.uint8)
    cap = len(data) // 2 + 2
    keys = np.full(cap, -7, np.int64)
    assert L.gccb_edgelist_begin(fmt, ptr(ws), ws_bytes, None) == 0
    reader = ChunkReader(io.BytesIO(data), chunk)
    buf = np.zeros(chunk, np.uint8)
    chunks = []
    while True:
        nb = reader.fill(buf)
        if nb == 0:
            break
        chunks.append(bytes(buf[:nb]))
        assert L.gccb_edgelist_parse(ptr(buf), nb, fmt, ptr(keys), cap, ptr(ws), ws_bytes, None) == 0
    assert b"".join(chunks) == data
    assert all(c.endswith(b"\n") for c in chunks[:-1])
    assert L.gccb_edgelist_finish(fmt, ptr(keys), ptr(ws), ws_bytes, None) == 0
    st = _capi.EdgelistState.from_buffer_copy(ws[:C.sizeof(_capi.EdgelistState)].tobytes())
    return st, keys[:st.keys], chunks


def check_against_oracle(data, fmt, chunk):
    st, keys, chunks = emu_parse(data, fmt, chunk)
    ref = oracle.parse_keys(data, fmt)
    err = None if st.first_error == NONE else (st.first_error >> 4, st.first_error & 15)
    assert err == ref["error"]
    if err is None:
        np.testing.assert_array_equal(keys, ref["keys"])
        assert st.n == ref["n"]
        assert st.edge_lines == ref["edge_lines"]
        assert st.lines == ref["lines"]
        if fmt == oracle.LSCC:
            assert st.m == ref["m"]
    return st, keys, chunks


SEPS = [b" ", b"  ", b"\t", b" \t ", b"\t\t"]


def _sep(rng):
    return SEPS[rng.integers(len(SEPS))]


def _line(rng, toks, eol):
    lead = b"" if rng.random() < 0.6 else _sep(rng)
    trail = b"" if rng.random() < 0.6 else _sep(rng)
    body = toks[0]
    for t in toks[1:]:
        body += _sep(rng) + t
    return lead + body + trail + eol


def make_lscc(rng, n, m, crlf=False, tail_newline=True, extra=2):
    eol = b"\r\n" if crlf else b"\n"
    out = [_line(rng, [b"n", b"%d" % n], eol)]
    out += [_line(rng, [b"%d" % i, b"v%d" % (i * 7)], eol) for i in range(n)]
    out.append(_line(rng, [b"m", b"%d" % m], eol))
    for _ in range(m):
        u, v = rng.integers(0, n, 2)
        if rng.random() < 0.1:
            v = u                                   # self loop
        out.append(_line(rng, [b"%d" % u, b"%d" % v, b"%d" % rng.integers(1, 9)], eol))
    out += [b"trailing line %d ignored" % k + eol for k in range(extra)]
    data = b"".join(out)
    return data if tail_newline else data.rstrip(b"\r\n")


def make_plain(rng, n, m, crlf=False, tail_newline=True):
    eol = b"\r\n" if crlf else b"\n"
    out = [b"# a SNAP-style header" + eol, b"% another comment" + eol]
    for k in range(m):
        r = rng.random()
        if r < 0.05:
            out.append(_sep(rng) + eol if rng.random() < 0.5 else eol)      # blank or whitespace-only line
        elif r < 0.08:
            out.append(_sep(rng) + b"# indented comment" + eol)
        u, v = rng.integers(0, n, 2)
        if rng.random() < 0.1:
            v = u
        toks = [b"%d" % u, b"%d" % v] + ([b"1.5", b"ts=3"] if rng.random() < 0.2 else [])
        out.append(_line(rng, toks, eol))
    data = b"".join(out)
    return data if tail_newline else data.rstrip(b"\r\n")


@pytest.mark.parametrize("chunk", [64, 200, 301])
@pytest.mark.parametrize("crlf,tail", [(False, True), (True, True), (False, False), (True, False)])
def test_lscc_keys_equal_restatement(chunk, crlf, tail):
    rng = np.random.default_rng(chunk * 4 + crlf * 2 + tail)
    data = make_lscc(rng, 23, 60, crlf=crlf, tail_newline=tail)
    st, keys, chunks = check_against_oracle(data, oracle.LSCC, chunk)
    assert len(chunks) >= 3 and st.keys > 0


@pytest.mark.parametrize("chunk", [64, 200, 301])
@pytest.mark.parametrize("crlf,tail", [(False, True), (True, True), (False, False), (True, False)])
def test_plain_keys_equal_restatement(chunk, crlf, tail):
    rng = np.random.default_rng(100 + chunk * 4 + crlf * 2 + tail)
    data = make_plain(rng, 40, 70, crlf=crlf, tail_newline=tail)
    st, keys, chunks = check_against_oracle(data, oracle.PLAIN, chunk)
    assert len(chunks) >= 3 and st.keys > 0


def test_chunk_boundaries_on_newlines():
    """16-byte lines and a 256-byte chunk: every full chunk ends exactly on '\\n' and carries nothing over."""
    lines = [b"n %13d\n" % 40] + [b"%7d %7d\n" % (i, i) for i in range(40)] + [b"m %13d\n" % 30]
    lines += [b"%4d %4d %5d\n" % (i % 40, (i * 7 + 1) % 40, 1) for i in range(30)]
    data = b"".join(lines)
    assert all(len(x) == 16 for x in lines)
    st, keys, chunks = check_against_oracle(data, oracle.LSCC, 256)
    assert all(len(c) == 256 for c in chunks[:-1])


def test_empty_plain_file():
    st, keys, _ = check_against_oracle(b"# nothing\n\n", oracle.PLAIN, 64)
    assert st.n == 0 and st.keys == 0


def _lscc_lines(edges, n=5, m=None):
    m = len(edges) if m is None else m
    return b"".join([b"n %d\n" % n] + [b"%d 0\n" % i for i in range(n)] + [b"m %d\n" % m] + [e + b"\n" for e in edges])


# (data, format, 1-based line, kind): every error names the first offending line
ERRORS = [
    (_lscc_lines([b"0 1 1", b"1 2", b"2 3 1"]), oracle.LSCC, 9, oracle.TOKENS),
    (_lscc_lines([b"0 1 1", b"1 2 1 4"]), oracle.LSCC, 9, oracle.TOKENS),
    (_lscc_lines([b"0 1 1", b"", b"2 3 1"]), oracle.LSCC, 9, oracle.TOKENS),
    (_lscc_lines([b"0 1 1", b"1 x 1"]), oracle.LSCC, 9, oracle.CHAR),
    (_lscc_lines([b"0 1 1", b"1 2 +1"]), oracle.LSCC, 9, oracle.CHAR),
    (_lscc_lines([b"0 1 1", b"1 5 1"]), oracle.LSCC, 9, oracle.RANGE),
    (_lscc_lines([b"0 -1 1", b"1 5 1"]), oracle.LSCC, 8, oracle.RANGE),
    (_lscc_lines([b"0 1 1", b"1 99999999999999999999 1"]), oracle.LSCC, 9, oracle.OVERFLOW),
    (_lscc_lines([b"0 1 1", b"1 2 1"], m=4), oracle.LSCC, 10, oracle.SHORT),
    (b"n 3\n0\n1\n", oracle.LSCC, 5, oracle.SHORT),
    (b"", oracle.LSCC, 1, oracle.SHORT),
    (b"n\n0\n", oracle.LSCC, 1, oracle.TOKENS),
    (b"n -4\n", oracle.LSCC, 1, oracle.RANGE),
    (b"# c\n0 1\n7\n2 3\n", oracle.PLAIN, 3, oracle.TOKENS),
    (b"0 1\n2 3x\n", oracle.PLAIN, 2, oracle.CHAR),
    (b"0 1\n-2 3\n", oracle.PLAIN, 2, oracle.RANGE),
    (b"0 1\n2 2147483648\n", oracle.PLAIN, 2, oracle.RANGE),
    (b"0 1\n2 -9223372036854775809\n", oracle.PLAIN, 2, oracle.OVERFLOW),
]


@pytest.mark.parametrize("data,fmt,line,kind", ERRORS)
def test_errors_name_the_line(data, fmt, line, kind):
    for chunk in (16, 64):
        if max((len(x) for x in data.split(b"\n")), default=0) >= chunk:
            continue
        st, _, _ = emu_parse(data, fmt, chunk)
        assert st.first_error != NONE
        assert ((st.first_error >> 4) + 1, st.first_error & 15) == (line, kind)
        assert st.error_flags >> kind & 1
        ref = oracle.parse_keys(data, fmt)["error"]
        assert (ref[0] + 1, ref[1]) == (line, kind)


def test_ignored_parts_are_not_errors():
    # .lscc: a self loop out of range and an overflowing weight (the reference never checks either), anything on
    # the vertex and trailing lines; plain: extra tokens of any shape
    data = _lscc_lines([b"9 9 1", b"0 1 99999999999999999999"]) + b"garbage\n"
    st, keys, _ = check_against_oracle(data, oracle.LSCC, 64)
    assert st.first_error == NONE and list(keys) == [1, 5]
    st, keys, _ = check_against_oracle(b"0 1 x y z\n", oracle.PLAIN, 64)
    assert st.first_error == NONE and list(keys) == [1, 2]


def test_line_longer_than_chunk():
    reader = ChunkReader(io.BytesIO(b"0 1\n" + b"1" * 40 + b" 2\n"), 32)
    buf = np.zeros(32, np.uint8)
    assert reader.fill(buf) == 4
    with pytest.raises(LineTooLong):
        reader.fill(buf)


def test_from_keys_device_equals_from_pairs_on_cpu():
    rng = np.random.default_rng(3)
    n = 50
    src, dst = rng.integers(0, n, 300), rng.integers(0, n, 300)
    src[:20] = dst[:20]                              # self loops
    src = np.concatenate([src, dst[:30]])            # duplicates in the other orientation
    dst = np.concatenate([dst, src[:30]])
    ref = synthetic.from_pairs(src, dst, n)
    keep = src != dst
    s, d = torch.from_numpy(src[keep]), torch.from_numpy(dst[keep])
    parts = [s * n + d, d * n + s]
    got = synthetic.from_keys_device(parts, n)
    assert parts == []
    np.testing.assert_array_equal(got.indptr.numpy(), ref.indptr)
    np.testing.assert_array_equal(got.indices.numpy(), ref.indices)
    assert got.num_nodes == ref.num_nodes and got.indices.dtype == torch.int32


def _golden_graphs():
    z = np.load(GOLDEN)
    return z, [(z["file%d" % i].item(), z["indptr%d" % i], z["indices%d" % i]) for i in range(int(z["count"]))]


def test_emu_parse_and_cleaning_equal_reference_x2dgl():
    """The reference's own yuxiao_kdd17_graph_to_dgl (under tests/golden/dgl_stub.py) on the fixture files."""
    z, graphs = _golden_graphs()
    assert list(z["graph_sizes"]) == [len(indptr) - 1 for _, indptr, _ in graphs]
    for fname, indptr, indices in graphs:
        data = z["text_" + fname].tobytes()
        st, keys, _ = emu_parse(data, oracle.LSCC, 128)
        assert st.first_error == NONE
        g = synthetic.from_keys_device(torch.from_numpy(keys.copy()), int(st.n))
        np.testing.assert_array_equal(g.indptr.numpy(), indptr)
        np.testing.assert_array_equal(g.indices.numpy(), indices)
