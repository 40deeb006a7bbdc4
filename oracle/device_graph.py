"""Model of the device walk graph: what every part of ``annb_device_graph_export`` must hold for a host graph.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  A numpy statement of the walk layout (DESIGN §3, the
``GraphDev`` / ``WideDev`` comments of ``annb_internal.h``) from the reference's pickle state (``Engine.get_graph()``)
and the code geometry (n_subvectors, code bytes).  ``expected`` returns, per part, the exact bytes and a mask of the
bytes a comparison checks:

* level-0 records, ``rec0_bytes`` each: slot j < count holds the link and, for rows of <= 128 bytes, the code row of
  that link at ``code_off0 + j * code_row``; slot j >= count holds link 0xFFFFFFFF and a zero code.  Wide rows hold
  links only.  **Masked**: the alignment padding between the last link and ``code_off0``, and after the last code slot
  (for wide rows: everything after the links).  A full derivation never writes those bytes (the buffer is a fresh
  cudaMalloc), a patch writes zeros, and no walk reads them.  Every link and code slot is checked, so a code written
  to the wrong slot, or a record scattered to the wrong id, lands on a checked byte.
* upper levels, level l from ``up_off[l]``: the nodes with level >= l in id order, each record
  ``[maxM record indices at l][pad][maxM codes, or node ids for wide rows][pad][u32 node id][u32 down][pad]``, down =
  the node's record index at l - 1 (its node id at l = 1).  The host assembles this buffer zero-filled and uploads it
  whole, so every byte is checked, padding included.
* labels by internal id; the deleted bitmap, ``(n + 31) // 32 + 1`` words with the trailing word zero.
* wide code matrix rows, ``up16(code_row)`` bytes each; the row padding is masked as in level 0 (the full derivation's
  2-D copy skips it, a patch writes zeros).
* own codes: every node's code row by internal id.
* the header (``annlite_b200._lib.GRAPH_HEADER_BYTES``): the geometry, ``ep_rec`` (the entry point's record at
  ``maxlevel``, its node id when ``maxlevel`` = 0, 0 for an empty graph), ``max_label`` / ``labels_identity``,
  ``up_off`` (0 above ``maxlevel``) and ``ep_code`` (the entry node's code for rows of <= 128 bytes, zero-padded to
  128 bytes; all zero for wide rows and an empty graph).  All checked.
"""
import numpy as np

NARROW_CODE_ROW = 128
MAX_LEVELS = 32
HEADER_FIELDS = ('n', 'maxlevel', 'ep_node', 'ep_rec', 'maxM', 'maxM0', 'code_row', 'rec0_bytes', 'code_off0',
                 'recu_bytes', 'code_offu', 'tail_offu', 'max_label', 'labels_identity')
HEADER_BYTES = (len(HEADER_FIELDS) + MAX_LEVELS) * 8 + 128
EMPTY = 0xFFFFFFFF


def up16(v):
    return (v + 15) // 16 * 16


def geometry(max_M, max_M0, code_row):
    """(rec0_bytes, code_off0, recu_bytes, code_offu, tail_offu, wide) as sync_device_graph lays them out."""
    wide = code_row > NARROW_CODE_ROW
    if wide:
        code_off0, rec0_bytes = 0, up16(4 * max_M0)
        code_offu = up16(4 * max_M)
        tail_offu = (code_offu + 4 * max_M + 7) // 8 * 8
    else:
        code_off0 = up16(4 * max_M0)
        rec0_bytes = up16(code_off0 + max_M0 * code_row)
        code_offu = up16(4 * max_M)
        tail_offu = (code_offu + max_M * code_row + 7) // 8 * 8
    return rec0_bytes, code_off0, up16(tail_offu + 8), code_offu, tail_offu, wide


def parse_header(buf):
    """Header bytes -> dict of its fields, with 'up_off' (32,) and 'ep_code' (128 bytes)."""
    buf = np.asarray(buf, dtype=np.uint8)
    assert buf.size == HEADER_BYTES, buf.size
    f = buf[:len(HEADER_FIELDS) * 8].view(np.int64)
    out = {k: int(v) for k, v in zip(HEADER_FIELDS, f)}
    o = len(HEADER_FIELDS) * 8
    out['up_off'] = buf[o:o + 8 * MAX_LEVELS].view(np.int64).copy()
    out['ep_code'] = buf[o + 8 * MAX_LEVELS:].copy()
    return out


class _State:
    """The parts of a pickle state the layout reads, as arrays."""

    def __init__(self, st, M_sub, code_bytes):
        self.n = int(st['cur_element_count'])
        self.maxlevel, self.ep = int(st['max_level']), int(st['enterpoint_node']) & EMPTY
        self.maxM, self.maxM0 = int(st['max_M']), int(st['max_M0'])
        self.code_row = int(M_sub) * int(code_bytes)
        spe, od, lo = int(st['size_data_per_element']), int(st['offset_data']), int(st['label_offset'])
        assert lo - od == self.code_row, 'code geometry does not match the state'
        r = np.asarray(st['data_level0']).view(np.uint8)[:self.n * spe].reshape(self.n, spe)
        self.count = np.ascontiguousarray(r[:, 0:2]).view(np.uint16).ravel().astype(np.int64)
        self.deleted = (r[:, 2] & 1).astype(bool)
        self.links = np.ascontiguousarray(r[:, 4:4 + 4 * self.maxM0]).view(np.uint32).reshape(self.n, self.maxM0)
        self.codes = np.ascontiguousarray(r[:, od:lo])
        self.labels = np.ascontiguousarray(r[:, lo:lo + 8]).view(np.uint64).ravel()
        self.levels = np.asarray(st['element_levels'], dtype=np.int64)[:self.n]
        self.slpe = int(st['size_links_per_element'])
        self.link_lists = np.asarray(st['link_lists']).view(np.uint8).ravel()
        self.link_off = np.concatenate([[0], np.cumsum(np.maximum(self.levels, 0) * self.slpe)[:-1]]).astype(np.int64) \
            if self.n else np.zeros(0, np.int64)

    def upper_list(self, u, l):
        """(count, links uint32 (maxM,)) of node u at level l >= 1"""
        o = self.link_off[u] + (l - 1) * self.slpe
        c = int(self.link_lists[o:o + 2].view(np.uint16)[0])
        return c, self.link_lists[o + 4:o + 4 + 4 * self.maxM].view(np.uint32)


def expected(st, M_sub, code_bytes):
    """part -> (bytes uint8, checked bool) for every part of the export; see the module docstring."""
    s = _State(st, M_sub, code_bytes)
    n, crow, M0, Mu = s.n, s.code_row, s.maxM0, s.maxM
    rec0_bytes, code_off0, recu_bytes, code_offu, tail_offu, wide = geometry(Mu, M0, crow)
    out = {}

    # level 0
    j = np.arange(M0)
    live = j[None, :] < s.count[:, None]
    links = np.where(live, s.links, np.uint32(EMPTY)).astype(np.uint32)
    rec = np.zeros((n, rec0_bytes), np.uint8)
    chk = np.zeros((n, rec0_bytes), bool)
    rec[:, :4 * M0] = links.view(np.uint8).reshape(n, 4 * M0)
    chk[:, :4 * M0] = True
    if not wide:
        nb = s.codes[np.where(live, s.links, 0).astype(np.int64)] if n else np.zeros((0, M0, crow), np.uint8)
        nb = np.where(live[:, :, None], nb, 0).astype(np.uint8)
        rec[:, code_off0:code_off0 + M0 * crow] = nb.reshape(n, M0 * crow)
        chk[:, code_off0:code_off0 + M0 * crow] = True
    out['rec0'] = (rec.ravel(), chk.ravel())

    # upper levels
    up_off = np.zeros(MAX_LEVELS, np.int64)
    parts, ep_rec = [], (s.ep if n else 0)
    prev = None
    off = 0
    for l in range(1, s.maxlevel + 1) if n else ():
        nodes = np.flatnonzero(s.levels >= l)
        cur = np.full(n, EMPTY, np.int64)
        cur[nodes] = np.arange(nodes.size)
        up_off[l] = off
        recs = np.zeros((nodes.size, recu_bytes), np.uint8)
        cnt = np.empty(nodes.size, np.int64)
        lk = np.empty((nodes.size, Mu), np.int64)
        for r, u in enumerate(nodes):
            c, ll = s.upper_list(u, l)
            cnt[r], lk[r] = c, ll
        livu = np.arange(Mu)[None, :] < cnt[:, None]
        tgt = np.where(livu, lk, 0)
        assert (cur[tgt][livu] != EMPTY).all(), 'a link to a node without level l'
        recs[:, :4 * Mu] = np.where(livu, cur[tgt], EMPTY).astype(np.uint32).view(np.uint8).reshape(-1, 4 * Mu)
        if wide:
            ids = np.where(livu, tgt, 0).astype(np.uint32)
            recs[:, code_offu:code_offu + 4 * Mu] = ids.view(np.uint8).reshape(-1, 4 * Mu)
        else:
            c = np.where(livu[:, :, None], s.codes[tgt], 0).astype(np.uint8)
            recs[:, code_offu:code_offu + Mu * crow] = c.reshape(-1, Mu * crow)
        down = nodes if l == 1 else prev[nodes]
        recs[:, tail_offu:tail_offu + 8] = np.stack([nodes, down], 1).astype(np.uint32).view(np.uint8).reshape(-1, 8)
        parts.append(recs.ravel())
        off += recs.size
        if l == s.maxlevel:
            ep_rec = int(cur[s.ep])
        prev = cur
    upper = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    out['upper'] = (upper, np.ones(upper.size, bool))

    out['labels'] = (s.labels.view(np.uint8).copy(), np.ones(8 * n, bool))
    words = np.zeros((n + 31) // 32 + 1, np.uint32)
    ids = np.flatnonzero(s.deleted)
    np.bitwise_or.at(words, ids >> 5, (np.uint32(1) << (ids & 31).astype(np.uint32)).astype(np.uint32))
    out['deleted'] = (words.view(np.uint8).copy(), np.ones(4 * words.size, bool))

    if wide:
        stride = up16(crow)
        wc = np.zeros((n, stride), np.uint8)
        wc[:, :crow] = s.codes
        wchk = np.zeros((n, stride), bool)
        wchk[:, :crow] = True
        out['wide_codes'] = (wc.ravel(), wchk.ravel())
    else:
        out['wide_codes'] = (np.zeros(0, np.uint8), np.zeros(0, bool))
    out['own_codes'] = (s.codes.ravel().copy(), np.ones(n * crow, bool))

    ep_code = np.zeros(128, np.uint8)
    if n and not wide:
        ep_code[:crow] = s.codes[s.ep]
    max_label = int(s.labels.max()) if n else 0
    max_label -= (1 << 64) if max_label >= 1 << 63 else 0     # the header's int64 holds the u64 bits
    ident = int(bool((s.labels == np.arange(n, dtype=np.uint64)).all()))
    f = [n, s.maxlevel, s.ep, ep_rec, Mu, M0, crow, rec0_bytes, code_off0, recu_bytes, code_offu, tail_offu,
         max_label, ident]
    head = np.concatenate([np.array(f, np.int64).view(np.uint8), up_off.view(np.uint8), ep_code])
    out['header'] = (head, np.ones(head.size, bool))
    return out


def mismatches(got, want):
    """Byte offsets where an exported part differs from the model on a checked byte (or a size message)."""
    v, chk = want
    got = np.asarray(got, dtype=np.uint8)
    if got.size != v.size:
        return f'{got.size} bytes, model {v.size}'
    return np.flatnonzero((got != v) & chk)
