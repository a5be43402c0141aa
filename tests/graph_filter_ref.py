"""CPU restatement of the WHERE-filtered graph hop and +collect (sdb_graph_expand_filtered / sdb_graph_collect_filtered),
written from the reference's semantics rather than the GPU design: the reference scans each source's edge keys in key
order, evaluates the hop's condition on every edge record (GraphScanOutput::FullEdge + Filter), keeps those that pass and
stops a source after `limit` kept ones.  Bitmaps: uint32 words, bit i = bit i % 32 of word i // 32 (None = no
condition)."""
import numpy as np


def bit(words, i):
    return (int(words[i >> 5]) >> (i & 31)) & 1


def bits_of(words, n):
    """the first n bits of a bitmap as a bool array"""
    b = np.unpackbits(np.ascontiguousarray(words, "<u4").view(np.uint8), bitorder="little")
    return b[:n].astype(bool)


def hop(row_ptr, col_idx, frontier, edge_bits=None, target_bits=None, limit=0):
    """one filtered hop: per source in frontier order, its passing targets in key (CSR) order, at most `limit` of them"""
    rp = np.asarray(row_ptr, np.int64)
    ci = np.asarray(col_idx, np.uint32)
    n_rows = rp.size - 1
    em = None if edge_bits is None else bits_of(edge_bits, ci.size)
    tm = None if target_bits is None else bits_of(target_bits, n_rows)
    out = []
    for v in np.asarray(frontier, np.int64):
        if v >= n_rows:
            raise IndexError(f"frontier id {v} out of range")
        b, e = rp[v], rp[v + 1]
        t = ci[b:e]
        keep = np.ones(e - b, bool)
        if em is not None:
            keep &= em[b:e]
        if tm is not None:
            keep &= tm[t]
        t = t[keep]
        out.append(t[:limit] if limit else t)
    return np.concatenate(out).astype(np.uint32) if out else np.zeros(0, np.uint32)


def chain(hops, frontier, limit=0):
    """hops: [(row_ptr, col_idx, edge_bits, target_bits), ...] applied in order"""
    fr = np.asarray(frontier, np.uint32)
    for rp, ci, eb, tb in hops:
        fr = hop(rp, ci, fr, eb, tb, limit)
    return fr


def collect(row_ptr, col_idx, start, edge_bits=None, target_bits=None, min_depth=1, max_depth=0, inclusive=False):
    """`.{min..max+collect[+inclusive]}` over the filtered hop: per BFS level the filtered hop of the frontier, first
    seen wins; the start values are emitted and marked seen only when inclusive (recursion/collect.rs)"""
    n_rows = np.asarray(row_ptr).size - 1
    seen = np.zeros(n_rows, bool)
    out = []
    frontier = [int(s) for s in start]
    if inclusive:
        for s in frontier:
            out.append(s)
            seen[s] = True
    depth = 0
    while frontier and (max_depth == 0 or depth < max_depth):
        nxt = []
        for t in hop(row_ptr, col_idx, frontier, edge_bits, target_bits):
            t = int(t)
            if seen[t]:
                continue
            seen[t] = True
            nxt.append(t)
        if depth + 1 >= min_depth:
            out += nxt
        frontier = nxt
        depth += 1
    return np.asarray(out, np.uint32)
