"""CPU: the device-graph layout model (oracle/device_graph.py) against a plain per-node restatement of DESIGN §3, on
the golden graph states and on host-only graphs at the geometries where the layout has padding, wide rows, many
levels, deletions at word edges, or no nodes at all."""
import numpy as np
import pytest

import oracle as O
from oracle import device_graph as DG
from annlite_b200 import _lib as L
from annlite_b200.engine import Engine
from conftest import CASES, Fixture

# (name, dim, n_subvectors, Ks, Mconn, n)
GEOMETRIES = [
    ('u8_m8', 32, 8, 256, 16, 300),          # maxM0 = 32: no padding in rec0
    ('u8_m5', 20, 5, 64, 10, 300),           # maxM0 = 20: 12 bytes of padding after the codes
    ('u16_m5', 20, 5, 400, 24, 300),         # two-byte codes, maxM0 = 48
    ('wide_u8_m192', 192, 192, 16, 5, 120),  # links-only records of 40 bytes in 48
    ('wide_u16_m72', 72, 72, 300, 5, 120),   # 144-byte code rows
    ('levels', 16, 4, 16, 2, 400),           # Mconn = 2: maxlevel >= 3
]


def loop_model(st, M_sub, code_bytes):
    """Every byte of every part, one node and one slot at a time, from DESIGN §3 / annb_internal.h."""
    n, M0, Mu = st['cur_element_count'], st['max_M0'], st['max_M']
    crow = M_sub * code_bytes
    wide = crow > 128
    spe, od = st['size_data_per_element'], st['offset_data']
    l0 = bytes(np.asarray(st['data_level0']).view(np.uint8)[:n * spe])
    ll = bytes(np.asarray(st['link_lists']).view(np.uint8))
    levels = [int(v) for v in np.asarray(st['element_levels'])[:n]]
    u16 = lambda b, o: int.from_bytes(b[o:o + 2], 'little')
    u32 = lambda b, o: int.from_bytes(b[o:o + 4], 'little')
    code = lambda u: l0[u * spe + od:u * spe + od + crow]
    label = lambda u: int.from_bytes(l0[u * spe + od + crow:u * spe + od + crow + 8], 'little')
    r16 = lambda v: (v + 15) // 16 * 16
    code_off0 = 0 if wide else r16(4 * M0)
    rec0_bytes = r16(4 * M0) if wide else r16(code_off0 + M0 * crow)
    code_offu = r16(4 * Mu)
    tail_offu = (code_offu + Mu * (4 if wide else crow) + 7) // 8 * 8
    recu_bytes = r16(tail_offu + 8)
    out = {}

    rec0, chk0 = bytearray(), []
    for u in range(n):
        r, c = bytearray(rec0_bytes), [False] * rec0_bytes
        cnt = u16(l0, u * spe)
        for j in range(M0):
            v = u32(l0, u * spe + 4 + 4 * j) if j < cnt else 0xFFFFFFFF
            r[4 * j:4 * j + 4] = v.to_bytes(4, 'little')
            c[4 * j:4 * j + 4] = [True] * 4
            if not wide:
                o = code_off0 + j * crow
                if j < cnt:
                    r[o:o + crow] = code(v)
                c[o:o + crow] = [True] * crow
        rec0 += r
        chk0 += c
    out['rec0'] = (rec0, chk0)

    # upper levels: record index of node u at level l = its rank among the nodes with level >= l
    maxlevel, ep = st['max_level'], int(st['enterpoint_node']) & 0xFFFFFFFF
    link_off, o = [], 0
    for u in range(n):
        link_off.append(o)
        o += max(levels[u], 0) * st['size_links_per_element']
    up, up_off, ep_rec = bytearray(), [0] * 32, (ep if n else 0)
    for l in range(1, maxlevel + 1) if n else ():
        nodes = [u for u in range(n) if levels[u] >= l]
        rank = {u: r for r, u in enumerate(nodes)}
        below = {u: r for r, u in enumerate(x for x in range(n) if levels[x] >= l - 1)}
        up_off[l] = len(up)
        for u in nodes:
            r = bytearray(recu_bytes)
            base = link_off[u] + (l - 1) * st['size_links_per_element']
            cnt = u16(ll, base)
            for j in range(Mu):
                if j < cnt:
                    v = u32(ll, base + 4 + 4 * j)
                    r[4 * j:4 * j + 4] = rank[v].to_bytes(4, 'little')
                    if wide:
                        r[code_offu + 4 * j:code_offu + 4 * j + 4] = v.to_bytes(4, 'little')
                    else:
                        r[code_offu + j * crow:code_offu + (j + 1) * crow] = code(v)
                else:
                    r[4 * j:4 * j + 4] = b'\xff\xff\xff\xff'
            down = u if l == 1 else below[u]
            r[tail_offu:tail_offu + 8] = u.to_bytes(4, 'little') + down.to_bytes(4, 'little')
            up += r
        if l == maxlevel:
            ep_rec = rank[ep]
    out['upper'] = (up, [True] * len(up))

    lab = b''.join(label(u).to_bytes(8, 'little') for u in range(n))
    out['labels'] = (lab, [True] * len(lab))
    words = [0] * ((n + 31) // 32 + 1)
    for u in range(n):
        if l0[u * spe + 2] & 1:
            words[u // 32] |= 1 << (u % 32)
    dl = b''.join(w.to_bytes(4, 'little') for w in words)
    out['deleted'] = (dl, [True] * len(dl))
    wc, wchk = bytearray(), []
    if wide:
        for u in range(n):
            wc += code(u) + bytes(r16(crow) - crow)
            wchk += [True] * crow + [False] * (r16(crow) - crow)
    out['wide_codes'] = (wc, wchk)
    own = b''.join(code(u) for u in range(n))
    out['own_codes'] = (own, [True] * len(own))

    labels = [label(u) for u in range(n)]
    max_label = max(labels) if n else 0
    head = [n, maxlevel, ep, ep_rec, Mu, M0, crow, rec0_bytes, code_off0, recu_bytes, code_offu, tail_offu,
            max_label, int(labels == list(range(n)))] + up_off
    hb = b''.join((v & (2 ** 64 - 1)).to_bytes(8, 'little') for v in head)
    hb += (code(ep) if n and not wide else b'') + bytes(128 - (crow if n and not wide else 0))
    out['header'] = (hb, [True] * len(hb))
    return out


def assert_models_agree(st, M_sub, code_bytes):
    vec, ref = DG.expected(st, M_sub, code_bytes), loop_model(st, M_sub, code_bytes)
    assert set(vec) == set(L.GRAPH_PARTS) == set(ref)
    for part in L.GRAPH_PARTS:
        v, c = vec[part]
        rv, rc = np.frombuffer(bytes(ref[part][0]), np.uint8), np.array(ref[part][1], bool)
        assert np.array_equal(c, rc), part
        assert np.array_equal(v[c], rv[rc]), part
    assert vec['header'][0].size == DG.HEADER_BYTES == L.GRAPH_HEADER_BYTES
    return vec


def host_graph(dim, M_sub, Ks, Mconn, n, seed=0, deleted=()):
    """A host-only handle with n rows inserted from their codes and tables (no GPU), and its pickle state."""
    rng = np.random.default_rng(seed)
    ds = dim // M_sub
    X = rng.standard_normal((max(n, Ks), dim)).astype(np.float32)
    cb = np.stack([X[rng.choice(len(X), Ks, replace=False), m * ds:(m + 1) * ds] for m in range(M_sub)])
    e = Engine(dim, M_sub, Ks, 'euclidean', device=-1)
    e.init_graph(max(n, 1), M=Mconn, ef_construction=24, random_seed=7)
    for s in range(0, n, 64):        # chunks keep the (rows, M, Ks) tables small
        rows = X[s:min(n, s + 64)]
        e.add_items_with_tables(O.encode(rows, cb), O.adc_table(rows, cb), np.arange(s, s + len(rows), dtype=np.uint64) * 3 + 1,
                                num_threads=1)
    for i in deleted:
        e.mark_deleted(int(i) * 3 + 1)
    return e, e.get_graph()


@pytest.mark.parametrize('name', CASES)
def test_model_on_golden_states(name):
    fx = Fixture(name)
    vec = assert_models_agree(fx.state, fx.M, 1 if fx.Ks <= 256 else 2)
    h = DG.parse_header(vec['header'][0])
    assert h['n'] == fx.state['cur_element_count'] and h['maxlevel'] == fx.state['max_level']


@pytest.mark.parametrize('geo', GEOMETRIES, ids=[g[0] for g in GEOMETRIES])
def test_model_on_host_built_graphs(geo):
    name, dim, M_sub, Ks, Mconn, n = geo
    e, st = host_graph(dim, M_sub, Ks, Mconn, n, deleted=(31, 32, 63, n - 1))
    cbytes = 1 if Ks <= 256 else 2
    vec = assert_models_agree(st, M_sub, cbytes)
    h = DG.parse_header(vec['header'][0])
    rec0_bytes, code_off0, recu_bytes, code_offu, tail_offu, wide = DG.geometry(st['max_M'], st['max_M0'], M_sub * cbytes)
    assert (h['rec0_bytes'], h['code_off0'], wide) == (rec0_bytes, code_off0, M_sub * cbytes > 128)
    # the geometry each case is here for
    if name == 'u8_m5':
        assert rec0_bytes > code_off0 + st['max_M0'] * M_sub          # padding after the codes
    if name.startswith('wide'):
        assert wide and rec0_bytes > 4 * st['max_M0']                  # padding after the links
    if name == 'levels':
        assert st['max_level'] >= 3
    words = DG.expected(st, M_sub, cbytes)['deleted'][0].view(np.uint32)
    assert words[0] >> 31 == 1 and words[1] & 3 == 1 and words[1] >> 31 == 1 and words[-1] == 0
    # the masks cover exactly the padding: every link and code slot is checked
    v, c = vec['rec0']
    c = c.reshape(n, rec0_bytes)
    assert c[:, :4 * st['max_M0']].all() and (c.sum(1) == 4 * st['max_M0'] + (0 if wide else st['max_M0'] * M_sub * cbytes)).all()


@pytest.mark.parametrize('n', [0, 1])
@pytest.mark.parametrize('M_sub,Ks', [(8, 256), (192, 16)])
def test_model_on_empty_and_single_node_graphs(n, M_sub, Ks):
    e, st = host_graph(M_sub * 2 if M_sub == 8 else M_sub, M_sub, Ks, 4, n)
    vec = assert_models_agree(st, M_sub, 1)
    h = DG.parse_header(vec['header'][0])
    assert h['n'] == n and h['max_label'] == (1 if n else 0) and h['labels_identity'] == (0 if n else 1)
    assert vec['rec0'][0].size == n * h['rec0_bytes'] and vec['upper'][0].size == 0
    assert vec['deleted'][0].size == 4 * ((n + 31) // 32 + 1) and not vec['deleted'][0].any()
    if n == 0:
        assert h['ep_rec'] == 0 and h['ep_node'] == 0xFFFFFFFF and not h['ep_code'].any()


def test_model_sees_a_code_in_the_wrong_slot_and_a_stale_record():
    """The masks leave no link or code slot unchecked: swapping two neighbour codes of one record, or one record for
    another, is a checked mismatch."""
    e, st = host_graph(32, 8, 256, 16, 200)
    vec = DG.expected(st, 8, 1)
    rec = vec['rec0'][0].reshape(200, -1).copy()
    h = DG.parse_header(vec['header'][0])
    o, crow = h['code_off0'], 8
    bad = rec.copy()
    bad[5, o:o + crow], bad[5, o + crow:o + 2 * crow] = rec[5, o + crow:o + 2 * crow], rec[5, o:o + crow]
    assert len(DG.mismatches(bad.ravel(), vec['rec0'])) > 0
    bad = rec.copy()
    bad[7] = rec[8]
    assert len(DG.mismatches(bad.ravel(), vec['rec0'])) > 0
    assert len(DG.mismatches(rec.ravel(), vec['rec0'])) == 0
