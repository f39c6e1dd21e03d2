"""Host restatements of the corpus builder (test infrastructure, not product):

  * parse_keys: csrc/edgelist.cu's parse, line by line in Python -- the keys in file order, the state fields and
    the first error -- for the emulator tests;
  * host_build: numpy parse + synthetic.from_pairs, the host path the GPU build is compared with at size.
"""
import numpy as np

from gcc_b200.datasets import synthetic

TOKENS, CHAR, RANGE, OVERFLOW, SHORT = 1, 2, 3, 4, 5
LSCC, PLAIN = 0, 1
I64_MAX = (1 << 63) - 1


def _int(tok):
    """-?[0-9]+ within int64 -> (value, error)."""
    body = tok[1:] if tok[:1] == b"-" else tok
    if not body or not all(48 <= c <= 57 for c in body):
        return None, CHAR
    v = int(tok)
    if v > I64_MAX or v < -I64_MAX - 1:
        return None, OVERFLOW
    return v, 0


def _tokens(line):
    return line.replace(b"\t", b" ").replace(b"\r", b" ").split(b" ")


def split_lines(data):
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    return lines


def parse_keys(data, fmt):
    """-> dict(keys, n, m, edge_lines, error=(0-based line, kind) or None)."""
    lines = split_lines(data)
    errors = []
    keys, edge_lines = [], 0
    n = m = -1
    if fmt == LSCC:
        def header(i):
            if i >= len(lines):
                errors.append((i, SHORT))
                return -2
            toks = [t for t in _tokens(lines[i]) if t]
            if len(toks) < 2:
                errors.append((i, TOKENS))
                return -2
            v, e = _int(toks[1])
            if not e and not 0 <= v < (1 << 31):
                e = RANGE
            if e:
                errors.append((i, e))
                return -2
            return v
        n = header(0)
        if n >= 0:
            m = header(n + 1)
        if n >= 0 and m >= 0:
            for i in range(n + 2, n + 2 + m):
                if i >= len(lines):
                    errors.append((i, SHORT))
                    break
                edge_lines += 1
                toks = [t for t in _tokens(lines[i]) if t]
                vals, err = [], 0
                for k, t in enumerate(toks[:3]):
                    v, e = _int(t)
                    if e == OVERFLOW and k == 2:
                        e, v = 0, 0
                    err = err or e
                    vals.append(v)
                if not err and len(toks) != 3:
                    err = TOKENS
                if err:
                    errors.append((i, err))
                    continue
                u, w = vals[0], vals[1]
                if u == w:
                    continue
                if not (0 <= u < n and 0 <= w < n):
                    errors.append((i, RANGE))
                    continue
                a, b = min(u, w), max(u, w)
                keys += [a * n + b, b * n + a]
    else:
        pairs = []
        for i, line in enumerate(lines):
            toks = [t for t in _tokens(line) if t]
            if not toks or toks[0][:1] in (b"#", b"%"):
                continue
            edge_lines += 1
            vals, err = [], 0
            for t in toks[:2]:
                v, e = _int(t)
                err = err or e
                vals.append(v)
            if not err and len(toks) < 2:
                err = TOKENS
            if err:
                errors.append((i, err))
                continue
            u, w = vals
            if u == w:
                continue
            if not (0 <= u < (1 << 31) and 0 <= w < (1 << 31)):
                errors.append((i, RANGE))
                continue
            pairs.append((min(u, w), max(u, w)))
        n = max([b for _, b in pairs], default=-1) + 1
        for a, b in pairs:
            keys += [a * n + b, b * n + a]
    return dict(keys=np.array(keys, dtype=np.int64), n=n, m=m, edge_lines=edge_lines, lines=len(lines),
                error=min(errors) if errors else None)


def _ints(body, width, piece=64 << 20):
    """Whitespace-separated integers of `body` as rows of `width`, parsed in pieces of about `piece` bytes."""
    out, pos = [], 0
    while pos < len(body):
        end = body.find(b"\n", min(pos + piece, len(body)))
        end = len(body) if end < 0 else end + 1
        out.append(np.array(body[pos:end].split(), dtype=np.int64))
        pos = end
    return (np.concatenate(out) if out else np.zeros(0, np.int64)).reshape(-1, width)


def host_pairs(path):
    """numpy parse of a well-formed file: (src, dst, n) of its edge lines, self loops included."""
    data = open(path, "rb").read()
    if str(path).endswith(".lscc"):
        head, _, rest = data.partition(b"\n")
        n = int(head.split()[1])
        parts = rest.split(b"\n", n + 1)
        m = int(parts[n].split()[1])
        body = parts[n + 1] if len(parts) > n + 1 else b""
        del data, rest, parts
        e = _ints(body, 3)[:m]
        return e[:, 0], e[:, 1], n
    if b"#" in data or b"%" in data:
        data = b"\n".join(ln for ln in data.split(b"\n") if ln.strip()[:1] not in (b"#", b"%"))
    e = _ints(data, 2)
    keep = e[:, 0] != e[:, 1]
    return e[:, 0], e[:, 1], int(e[keep].max()) + 1 if keep.any() else 0


def host_build(path, name="graph"):
    src, dst, n = host_pairs(path)
    return synthetic.from_pairs(src, dst, n, name)
