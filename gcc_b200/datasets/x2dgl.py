"""Pretraining corpus builder: raw edge-list files -> the ``.bin`` corpus that ``train.py --dataset <file>.bin``
reads.  The reference's gcc/utils/x2dgl.py, with the text parse on the GPU (csrc/edgelist.cu) and the cleaning
of x2dgl.py:52-62 in ``synthetic.from_keys_device``.

    python -m gcc_b200.datasets.x2dgl --graph-dir DIR --save-file FILE [--embed-dim N] [--graph-files F ...]

``--graph-dir`` takes the reference's six KDD'17 ``.lscc`` files (x2dgl.py:88-97) that are present in DIR;
``--graph-files`` adds other files: ``.lscc`` by suffix, anything else is read as a plain edge list ("u v" per
line, '#' / '%' comments).  ``--embed-dim`` is accepted and unused, as in the reference.
"""
import argparse
import ctypes
import logging
import os
import pathlib

import numpy as np
import torch

from .. import _capi, _lib
from . import dgl_bin, synthetic

logger = logging.getLogger(__name__)

TODO = ("ca-DBLP-NetRep.txt.lpm.lscc", "ca-DBLP-SNAP.txtu.lpm.lscc", "ca-IMDB-NetRep.txt.lpm.lscc",
        "soc-Academia-NetRep.txt.lpm.lscc", "soc-LiveJournal1-d-SNAP.txtu.lpm.lscc",
        "soc-Facebook1-NetRep.txt.lpm.lscc")
DEFAULT_CHUNK = 32 << 20


def file_format(path):
    return _capi.EL_LSCC if str(path).endswith(".lscc") else _capi.EL_PLAIN


class LineTooLong(Exception):
    pass


class ChunkReader:
    """Fills staging buffers of `cap` bytes with whole lines of a binary file: each chunk is cut after its last
    '\\n' and the rest goes to the front of the next one.  The file's last chunk may end without a newline."""

    def __init__(self, f, cap):
        self.f, self.cap, self.tail = f, cap, b""

    def fill(self, buf):
        """buf: writable uint8 array of `cap` bytes.  Returns the chunk's length (0 at the end of the file);
        raises LineTooLong when `cap` bytes hold no newline."""
        t = len(self.tail)
        buf[:t] = np.frombuffer(self.tail, dtype=np.uint8)
        got = t
        while got < self.cap:                       # a short read is not the end of the file
            r = self.f.readinto(memoryview(buf)[got:])
            if not r:
                break
            got += r
        if got < self.cap:                          # end of file: everything goes
            self.tail = b""
            return got
        win = 4096
        while True:
            lo = max(0, got - win)
            cut = bytes(buf[lo:got]).rfind(b"\n")
            if cut >= 0:
                cut += lo + 1
                break
            if lo == 0:
                raise LineTooLong()
            win *= 4
        self.tail = bytes(buf[cut:got])
        return cut


def _raise_error(path, st):
    fe = int(st.first_error)
    raise _lib.GccbError("%s:%d: %s" % (path, (fe >> 4) + 1, _capi.EL_ERR_NAMES.get(fe & 15, "parse error")))


def build_graph(path, chunk_bytes=DEFAULT_CHUNK):
    """One raw file -> CSRGraph on the current CUDA device, cleaned as x2dgl.py:40-62 cleans it.  The file is read
    in chunks of `chunk_bytes` into two pinned buffers; the copy of one chunk to the device (one stream) overlaps
    the parse of the other (a second stream) and the disk read of the next.  Logs the reference's figures
    (x2dgl.py:49,63-69).  Raises GccbError naming the file and line of malformed input, and before allocating when
    the keys and the de-duplication do not fit in free device memory."""
    _lib.require_device()
    lib = _lib.get()
    path = str(path)
    fmt = file_format(path)
    logger.info("processing %s", path)
    size = os.path.getsize(path)
    chunk_bytes = int(chunk_bytes)
    # an edge line that yields two keys holds at least "u v\n" (4 bytes; 3 for the file's last line)
    cap = size // 2 + 2
    ws_bytes = lib.gccb_edgelist_workspace(chunk_bytes)
    need = 8 * cap + 3 * 8 * cap + ws_bytes + 2 * chunk_bytes   # keys, then torch.unique's sort and output
    free = torch.cuda.mem_get_info()[0] + torch.cuda.memory_reserved() - torch.cuda.memory_allocated()
    if need > free:
        raise _lib.GccbError("%s: building needs %.2f GB of device memory (%.2f GB of keys, %.2f GB for their "
                             "de-duplication, %.2f GB of staging), %.2f GB are free; graphs that do not fit are "
                             "not supported" % (path, need / 1e9, 8 * cap / 1e9, 24 * cap / 1e9,
                                                (ws_bytes + 2 * chunk_bytes) / 1e9, free / 1e9))
    dev = torch.device("cuda", torch.cuda.current_device())
    keys = torch.empty(cap, dtype=torch.int64, device=dev)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    text = [torch.empty(chunk_bytes, dtype=torch.uint8, device=dev) for _ in range(2)]
    pinned = [torch.empty(chunk_bytes, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    host = [p.numpy() for p in pinned]
    copied = [torch.cuda.Event() for _ in range(2)]
    parsed = [torch.cuda.Event() for _ in range(2)]
    copy_s, parse_s = torch.cuda.Stream(), torch.cuda.Stream()
    parse_s.wait_stream(torch.cuda.current_stream())        # the buffers above were allocated on it
    copy_s.wait_stream(torch.cuda.current_stream())
    sp = ctypes.c_void_p(parse_s.cuda_stream)
    _lib.check(lib.gccb_edgelist_begin(fmt, _lib.dptr(ws), ws_bytes, sp), "gccb_edgelist_begin")

    def state():
        with torch.cuda.stream(parse_s):
            raw = ws[:ctypes.sizeof(_capi.EdgelistState)].cpu()
        parse_s.synchronize()
        return _capi.EdgelistState.from_buffer_copy(raw.numpy().tobytes())

    with open(path, "rb", buffering=0) as f:
        reader = ChunkReader(f, chunk_bytes)
        i = 0
        while True:
            s = i & 1
            copied[s].synchronize()                 # pinned[s] is free once its last copy has run
            try:
                nb = reader.fill(host[s])
            except LineTooLong:
                raise _lib.GccbError("%s:%d: line longer than the %d-byte staging chunk" % (
                    path, state().lines + 1, chunk_bytes)) from None
            if nb == 0:
                break
            with torch.cuda.stream(copy_s):
                copy_s.wait_event(parsed[s])        # text[s] is free once the parse of chunk i-2 has run
                text[s][:nb].copy_(pinned[s][:nb], non_blocking=True)
                copied[s].record(copy_s)
            parse_s.wait_event(copied[s])
            _lib.check(lib.gccb_edgelist_parse(_lib.dptr(text[s]), nb, fmt, _lib.dptr(keys), cap, _lib.dptr(ws),
                                               ws_bytes, sp), "gccb_edgelist_parse")
            parsed[s].record(parse_s)
            i += 1
    _lib.check(lib.gccb_edgelist_finish(fmt, _lib.dptr(keys), _lib.dptr(ws), ws_bytes, sp), "gccb_edgelist_finish")
    st = state()
    if st.first_error != (1 << 64) - 1:
        _raise_error(path, st)
    torch.cuda.current_stream().wait_stream(parse_s)
    del ws, text, pinned, host
    n, m = int(st.n), int(st.m if fmt == _capi.EL_LSCC else st.edge_lines)
    m_true = int(st.keys)
    logger.info("raw file has %d nodes and %d edges", n, m)
    parts = [keys[:m_true]]
    del keys
    g = synthetic.from_keys_device(parts, n, os.path.basename(path))
    logger.info("%d nodes, %d edges, %d self-loop(s) removed, %d zero-degree node(s) removed",
                g.num_nodes, len(g.indices), 2 * m - m_true, n - g.num_nodes)
    return g


def build_corpus(files, save_file):
    """x2dgl.py:99-131: every file built, the graphs sorted by vertex count, largest first (a stable sort, so
    ties keep the order of `files`), written with a "graph_sizes" label.  Returns the host graphs as written."""
    graphs = []
    for f in files:
        g = build_graph(f)
        graphs.append(synthetic.CSRGraph(g.indptr.cpu().numpy(), g.indices.cpu().numpy(), g.num_nodes, g.name))
        del g
    graphs.sort(key=lambda g: g.num_nodes, reverse=True)
    for i, g in enumerate(graphs):
        print(i, "%s: %d nodes, %d edges" % (g.name, g.num_nodes, len(g.indices)), g.num_nodes)
    logger.info("save graphs to %s", save_file)
    dgl_bin.write_dgl_bin(save_file, graphs)
    return graphs


def main(argv=None):
    parser = argparse.ArgumentParser("argument for x2dgl")
    parser.add_argument("--graph-dir", type=str, required=True, help="dir to load graphs")
    parser.add_argument("--save-file", type=str, required=True, help="file to save graphs")
    parser.add_argument("--embed-dim", type=int, default=None, help="embeding dimension (unused)")
    parser.add_argument("--graph-files", type=str, nargs="*", default=[],
                        help="more files: .lscc by suffix, anything else a plain edge list")
    args = parser.parse_args(argv)
    logging.basicConfig(format="%(asctime)s - %(levelname)s - %(name)s - %(message)s",
                        datefmt="%m/%d/%Y %H:%M:%S", level=logging.INFO)
    graph_dir = pathlib.Path(args.graph_dir)
    files = sorted(p for p in graph_dir.iterdir() if p.is_file() and p.name in TODO) + \
        [pathlib.Path(f) for f in args.graph_files]
    if not files:
        parser.error("no input graphs: none of the reference's files is in %s and --graph-files is empty" % graph_dir)
    build_corpus(files, args.save_file)


if __name__ == "__main__":
    main()
