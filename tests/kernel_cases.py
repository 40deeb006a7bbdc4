"""Every CUDA kernel entry of libannlite_b200.so, by key, and which test is answerable for it.

A key is a kernel's demangled name reduced to `name<args>`: no return type, namespace or parameter list; integer and
bool template arguments as plain integers (`(int)16` -> 16, `(bool)1` / `true` -> 1), type arguments as short names
(`unsigned char` -> u8).  `library_keys()` reads them from the built library (cuobjdump -symbols | cu++filt), and
`test_gpu_instances.captured_keys` reduces the kernel names the CUDA profiler records with the same `kernel_key`.

Each key is in exactly one of two groups:
  COVERED      keys that some GPU case of tests/test_gpu_instances.py (CASES below) asserts it launched;
  ELSEWHERE    key -> the existing test that runs it (kernels off the search and scan paths).
tests/test_kernel_inventory.py asserts that the two groups partition the library's keys exactly."""
import os
import re
import shutil
import subprocess

_TYPES = {'unsigned char': 'u8', 'unsigned short': 'u16', 'unsigned int': 'u32', 'unsigned long': 'u64',
          'unsigned long long': 'u64', 'signed char': 'i8', 'char': 'i8', 'short': 'i16', 'int': 'i32',
          'long': 'i64', 'long long': 'i64', 'float': 'f32', 'double': 'f64', 'bool': 'b'}


def _split_top(s, sep=','):
    """split at `sep` outside <> and ()"""
    out, depth, cur = [], 0, ''
    for ch in s:
        if ch in '<(':
            depth += 1
        elif ch in '>)':
            depth -= 1
        if ch == sep and depth == 0:
            out.append(cur)
            cur = ''
        else:
            cur += ch
    out.append(cur)
    return out


def _arg(a):
    a = a.strip()
    m = re.fullmatch(r'\((?:int|unsigned int|long|unsigned long|short|char|unsigned char|bool)\)\s*(-?\d+)[uUlL]*', a)
    if m:
        return str(int(m.group(1)))
    if re.fullmatch(r'-?\d+[uUlL]*', a):
        return str(int(re.sub(r'[uUlL]+$', '', a)))
    if a in ('true', 'false'):
        return '1' if a == 'true' else '0'
    return _TYPES.get(a, a)


def kernel_key(name):
    """'void <unnamed>::hnsw_walk4<(int)16, (int)16, (bool)0>(GraphDev, SearchParams)' -> 'hnsw_walk4<16,16,0>';
    also takes the profiler's form ('void (anonymous namespace)::hnsw_walk4<16, 16, false>(GraphDev, SearchParams)')."""
    s = name.strip()
    s = re.sub(r'^void\s+', '', s)
    s = s.replace('(anonymous namespace)::', '').replace('<unnamed>::', '').replace('{anonymous}::', '')
    # cut the parameter list: the first '(' at template depth 0 that is not a cast inside <...>
    depth, cut = 0, len(s)
    for i, ch in enumerate(s):
        if ch == '<':
            depth += 1
        elif ch == '>':
            depth -= 1
        elif ch == '(' and depth == 0:
            cut = i
            break
    s = s[:cut].strip()
    s = s.split('::')[-1] if '<' not in s else s[:s.index('<')].split('::')[-1] + s[s.index('<'):]
    if '<' not in s:
        return s
    base, args = s[:s.index('<')], s[s.index('<') + 1:s.rindex('>')]
    return base + '<' + ','.join(_arg(a) for a in _split_top(args)) + '>'


def _tool(name):
    p = shutil.which(name)
    if p:
        return p
    p = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', name)
    return p if os.path.exists(p) else None


def library_keys(path):
    """the keys of every kernel entry (STO_ENTRY) in the device code of `path`"""
    dump = subprocess.run([_tool('cuobjdump'), '-symbols', path], check=True, capture_output=True, text=True).stdout
    names = [ln.split('STO_ENTRY', 1)[1].strip() for ln in dump.splitlines() if 'STO_ENTRY' in ln]
    dem = subprocess.run([_tool('cu++filt')], input='\n'.join(names) + '\n', check=True, capture_output=True,
                         text=True).stdout.splitlines()
    assert len(dem) == len(names)
    return {kernel_key(d) for d in dem}


# ---- graph geometries -------------------------------------------------------------------------------------------
# name -> dict(N, D, M, Ks, Mconn, dup).  code row = M bytes (Ks <= 256) or 2M (u16); maxM0 = 2 * Mconn (> 32: the
# chunked walk); M * Ks * 4 bytes of table above the 227 KB opt-in shared memory of an H100: read from global memory.
SMEM_OPTIN = 232448
GEOMS = {
    'u8m4': dict(N=3000, D=16, M=4, Ks=256, Mconn=16),
    'u8m6': dict(N=3000, D=24, M=6, Ks=256, Mconn=16),
    'u8m8': dict(N=4000, D=32, M=8, Ks=256, Mconn=16),
    'u8m16': dict(N=3000, D=64, M=16, Ks=256, Mconn=16),
    'u8m32': dict(N=3000, D=128, M=32, Ks=256, Mconn=16),
    'u16m4': dict(N=3000, D=16, M=4, Ks=700, Mconn=16),
    'u16m5': dict(N=3000, D=20, M=5, Ks=400, Mconn=16),
    'u16m8': dict(N=3000, D=32, M=8, Ks=300, Mconn=16),
    'big16m8': dict(N=3000, D=16, M=8, Ks=7400, Mconn=16),
    'big16m4': dict(N=3000, D=8, M=4, Ks=15000, Mconn=16),
    'big16m5': dict(N=3000, D=10, M=5, Ks=12000, Mconn=16),
    'dup8': dict(N=1200, D=32, M=8, Ks=256, Mconn=16, dup=3),
    'wide8': dict(N=3000, D=192, M=192, Ks=256, Mconn=16),
    'wide16': dict(N=3000, D=144, M=72, Ks=300, Mconn=16),
}
for _n in ['u8m4', 'u8m6', 'u8m8', 'u8m16', 'u8m32', 'u16m4', 'u16m5', 'u16m8', 'big16m8', 'big16m4', 'big16m5']:
    GEOMS[_n + 'c'] = dict(GEOMS[_n], Mconn=24)          # maxM0 = 48 > 32: the chunked walk


def code_bytes(g):
    return 1 if g['Ks'] <= 256 else 2


def code_row_kind(g):
    """the CR template argument the walk launchers dispatch on (0 = generic rows)"""
    cr = g['M'] * code_bytes(g)
    return cr if cr in ((4, 8, 16, 32) if code_bytes(g) == 1 else (8, 16)) else 0


def wide(g):
    return g['M'] * code_bytes(g) > 128


def smem_table(g, epl, general):
    extra = (32 * epl + (256 if general else (0 if g['Mconn'] > 16 else 33))) * 8
    return (g['M'] * g['Ks'] * 4 + 15) // 16 * 16 + extra <= SMEM_OPTIN


EPLS = (2, 4, 8, 16)


def efs_for(epl):
    """both ends of an EPL class: 16*EPL+1 and the exactly full list 32*EPL"""
    return 16 * epl + 1, 32 * epl


# ---- the cases -------------------------------------------------------------------------------------------------
# A case: id, kind, geometry, search options, runs, and the keys it claims.  A run is (ef, k) or (ef, k, sel): the
# filtered kinds admit a random fraction `sel` of the labels (the run's own, else the case's).
#   kind: 'plain' (Engine.search), 'filter' (filter_labels), 'multi' (search_multi, two prepared filters alternating
#         over the queries), 'cells' / 'cells_filter' / 'cells_qfilter' (CellSet.search), 'repeat' (64 queries x 64)
CASES = []


def _case(cid, kind, geom, opts, runs, keys, **kw):
    CASES.append(dict(id=cid, kind=kind, geom=geom, opts=dict(opts), runs=list(runs), keys=set(keys), **kw))


def _runs(epl):
    lo, hi = efs_for(epl)
    return [(lo, 1), (hi, 10), (hi, hi)]       # k = ef: the full list is output


def _flagged_runs(epl):
    """hnsw_walk_flagged with its list forced to CAP = 32*EPL entries keeps every evaluated node until ef of them pass
    the filter, and it tests for overflow before it merges a hop's candidates (up to maxM0 <= 32 of them) and trims
    what falls behind the ef-th passing entry; a query that would overflow is re-run on the bitmap walk.  So the
    largest list it always serves is ef = CAP - 32 under a filter that admits every label (the host, which sizes CAP
    >= 1.3 ef / selectivity + 48, never asks for more), and the filtered runs leave room for the rejected nodes too."""
    full = 32 * epl - 32
    return [(8 * epl, 10, 0.7), (24 * epl - 32, 1, 0.9), (full, 10, 1.0), (full, full, 1.0)]


_ROUND1 = ['u8m4', 'u8m6', 'u8m8', 'u8m16', 'u8m32', 'u16m4', 'u16m5', 'u16m8', 'big16m8', 'big16m4', 'big16m5']
for _g in _ROUND1 + [n + 'c' for n in _ROUND1]:
    G = GEOMS[_g]
    cr, cb = code_row_kind(G), code_bytes(G)
    chunked = G['Mconn'] > 16
    for epl in EPLS:
        fam = 'hnsw_walk_chunked' if chunked else 'hnsw_walk_fast'
        sm = int(smem_table(G, epl, False))
        _case(f'fast-{_g}-e{epl}', 'plain', _g, {'walk_kernel': 1}, _runs(epl), [f'{fam}<{epl},{cr},{cb},{sm}>'])
        if not chunked:      # one general case per (geometry, EPL, PQF): the chunked graphs repeat the same keys
            sm = int(smem_table(G, epl, True))
            _case(f'general-{_g}-e{epl}', 'plain', _g, {'force_general': 2}, _runs(epl),
                  [f'hnsw_walk_general<{epl},{cr},{cb},{sm},0>'])
            _case(f'generalq-{_g}-e{epl}', 'multi', _g, {'force_general': 2}, _runs(epl)[1:2],
                  [f'hnsw_walk_general<{epl},{cr},{cb},{sm},1>'], sel=0.5)
            if cr != 0 and smem_table(G, epl, False):
                _case(f'flagged-{_g}-e{epl}', 'filter', _g, {'flagged_kernel': 1, 'flagged_epl': epl}, _flagged_runs(epl),
                      [f'hnsw_walk_flagged<{epl},{cr},{cb},0>'])
                _case(f'flaggedq-{_g}-e{epl}', 'multi', _g, {'flagged_kernel': 1, 'flagged_epl': epl},
                      [(24 * epl - 32, 10, 0.9), _flagged_runs(epl)[-1]], [f'hnsw_walk_flagged<{epl},{cr},{cb},1>'])

for _m in (8, 16, 32):
    for epl in EPLS:
        _case(f'walk4-m{_m}-e{epl}', 'plain', f'u8m{_m}', {}, _runs(epl), [f'hnsw_walk4<{_m},{epl},0>'])
    _case(f'walk4-m{_m}-ef512', 'plain', f'u8m{_m}', {}, [(512, 512), (512, 10)], [f'hnsw_walk4<{_m},16,0>'])
    for ep, ens, efs in ((2, (2, 3, 4, 5, 6, 8), (33, 64)), (4, (4, 6, 8), (65, 128))):
        for en in ens:
            _case(f'walk4f-m{_m}-p{ep}n{en}', 'filter', f'u8m{_m}', {'flagged_en': en}, [(efs[0], 1), (efs[1], 10), (efs[1], efs[1])],
                  [f'hnsw_walk4f<{_m},{ep},{en},0,0>'], sel=0.8)
            _case(f'walk4fq-m{_m}-p{ep}n{en}', 'multi', f'u8m{_m}', {'flagged_en': en}, [(efs[1], 10)],
                  [f'hnsw_walk4f<{_m},{ep},{en},1,0>'], sel=0.8)

for epl in EPLS:
    _case(f'cells-e{epl}', 'cells', 'u8m8', {}, _runs(epl), [f'hnsw_walk4<8,{epl},1>'])
for ep, ens, efs in ((2, (2, 3, 4, 5, 6, 8), (33, 64)), (4, (4, 6, 8), (65, 128))):
    for en in ens:
        _case(f'cellsf-p{ep}n{en}', 'cells_filter', 'u8m8', {'flagged_en': en}, [(efs[0], 1), (efs[1], 10)],
              [f'hnsw_walk4f<8,{ep},{en},0,1>'], sel=0.8)
        _case(f'cellsq-p{ep}n{en}', 'cells_qfilter', 'u8m8', {'flagged_en': en}, [(efs[1], 10)],
              [f'hnsw_walk4f<8,{ep},{en},1,1>'], sel=0.8)

for _g, cb in (('wide8', 1), ('wide16', 2)):
    for epl in EPLS:
        _case(f'wide-{_g}-e{epl}', 'plain', _g, {}, _runs(epl), [f'hnsw_walk_wide<{epl},{cb},0>'])
        _case(f'wideq-{_g}-e{epl}', 'multi', _g, {}, _runs(epl)[1:2], [f'hnsw_walk_wide<{epl},{cb},1>'], sel=0.5)

# duplicated vectors: exact ties everywhere; one case per walk family on the same graph
_case('ties-walk4', 'plain', 'dup8', {}, [(64, 64), (512, 512)], ['hnsw_walk4<8,2,0>', 'hnsw_walk4<8,16,0>'])
_case('ties-fast', 'plain', 'dup8', {'walk_kernel': 1}, [(64, 64), (512, 512)],
      ['hnsw_walk_fast<2,8,1,1>', 'hnsw_walk_fast<16,8,1,1>'])
_case('ties-general', 'plain', 'dup8', {'force_general': 2}, [(64, 64), (512, 512)],
      ['hnsw_walk_general<2,8,1,1,0>', 'hnsw_walk_general<16,8,1,1,0>'])
_case('ties-flagged', 'filter', 'dup8', {'flagged_kernel': 1, 'flagged_epl': 16}, [(64, 64, 0.7), (480, 480, 1.0)],
      ['hnsw_walk_flagged<16,8,1,0>'])
_case('ties-walk4f', 'filter', 'dup8', {'flagged_en': 3}, [(64, 64), (128, 128)], ['hnsw_walk4f<8,2,3,0,0>', 'hnsw_walk4f<8,4,4,0,0>'], sel=0.8)

# state carried from one query to the next on a warp: 64 queries x 64 repeats, with the default launch geometry and with
# one warp per CTA and one CTA per SM.  hnsw_walk_wide's launcher has a fixed CTA shape and ignores both options: there
# the repeats check the state its warps carry from query to query and the per-warp scratch reused across launches.
for fam, geom, opts, kind, ef, keys in (
        ('walk4', 'u8m8', {}, 'plain', 100, ['hnsw_walk4<8,4,0>']),
        ('walk4f', 'u8m8', {}, 'filter', 100, ['hnsw_walk4f<8,4,4,0,0>']),
        ('fast', 'u8m8', {'walk_kernel': 1}, 'plain', 100, ['hnsw_walk_fast<4,8,1,1>']),
        ('chunked', 'u8m8c', {'walk_kernel': 1}, 'plain', 100, ['hnsw_walk_chunked<4,8,1,1>']),
        ('flagged', 'u8m8', {'flagged_kernel': 1}, 'filter', 100, ['hnsw_walk_flagged<8,8,1,0>']),
        ('general-filter', 'u8m8', {'force_general': 2}, 'filter', 100, ['hnsw_walk_general<4,8,1,1,0>']),
        ('general-deleted', 'u8m8', {'force_general': 2}, 'deleted', 100, ['hnsw_walk_general<4,8,1,1,0>']),
        ('wide-filter', 'wide8', {}, 'filter', 100, ['hnsw_walk_wide<4,1,0>']),
        ('wide-deleted', 'wide8', {}, 'deleted', 100, ['hnsw_walk_wide<4,1,0>'])):
    _case(f'repeat-{fam}', 'repeat', geom, opts, [(ef, 10)], keys, inner=kind, sel=0.7)

# scans (ids and bits against oracle.scan_topk / oracle.scan) and the K1 table kernel
SCAN_K = (1, 33, 100, 200, 257, 512)
for _cb in (1, 2):
    for k in SCAN_K:
        epl = next(e for e in (1, 2, 4, 8, 16) if 32 * e >= k)
        _case(f'scan_topk-u{8 * _cb}-k{k}', 'scan_topk', None, {'scan_kernel': 1}, [(0, k)],
              [f'scan_topk_kernel<{epl},u{8 * _cb}>', 'merge_topk_kernel<u32,i64,1>'], cb=_cb)
for k, kk in ((1, 1), (10, 10), (16, 16)):
    _case(f'scan_tiled2-k{k}', 'scan_topk', None, {'scan_kernel': 2}, [(0, k)], [f'scan_topk_tiled2_kernel<{kk}>'], cb=1, M=8)
    _case(f'scan_tiled-k{k}', 'scan_topk', None, {'scan_kernel': 3}, [(0, k)], [f'scan_topk_tiled_kernel<{kk}>'], cb=1, M=8)
for _cb in (1, 2):
    _case(f'scan-u{8 * _cb}-smem', 'scan', None, {}, [], [f'scan_kernel<u{8 * _cb}>'], cb=_cb, Ks=256 if _cb == 1 else 300, M=8)
    _case(f'scan-u{8 * _cb}-global', 'scan', None, {}, [], [f'scan_kernel<u{8 * _cb}>'], cb=_cb, Ks=256 if _cb == 1 else 4000, M=128 if _cb == 1 else 32)    # table > 96 KB: read from global memory
ADC_DS = (0, 2, 4, 6, 8, 12, 16, 24, 32)
for ds in ADC_DS:
    _case(f'adc-ds{ds}', 'adc', None, {}, [], [f'adc_table_kernel<{ds}>'], ds=ds if ds else 5)
for k, e in ((1, 1), (10, 1), (16, 1), (20, 1), (33, 2), (100, 4), (200, 8), (257, 16), (512, 16)):
    _case(f'subset-k{k}', 'cells_bruteforce', 'u8m8', {}, [(k, k)],
          [f'subset_scan_tiled_kernel<{k if k in (1, 10, 16) else 16}>' if k <= 16 else f'subset_scan_warp_kernel<{e}>',
           'subset_gather_kernel'])
for G in (1, 2, 3, 8):
    _case(f'merge-G{G}', 'merge', None, {}, [], ['merge_sorted_kernel'], G=G)

COVERED = set().union(*(c['keys'] for c in CASES))

# ---- kernels of other paths and the tests that run them -------------------------------------------------------------
ELSEWHERE = {
    'encode_kernel<u8>': 'tests/test_gpu_parity.py (encode against oracle.encode); tests/test_gpu_build_model.py (built codes)',
    'encode_kernel<u16>': 'tests/test_gpu_wide_codes.py (u16 codes encoded on the device)',
    'l2_normalize_kernel': 'tests/test_gpu_parity.py (cosine queries normalised on the device)',
    'pack_rec0_kernel': 'tests/test_gpu_shapes.py (every search after set_graph / add_items)',
    'scatter_records_kernel': 'tests/test_gpu_build.py (incremental device-graph patches)',
    'mark_labels_kernel': 'tests/test_gpu_walk4f.py (filter_labels -> bitmap)',
    'gather_filter_kernel': 'tests/test_gpu_walk4f.py (filter_labels -> bitmap)',
    'export_links_kernel': 'tests/test_gpu_build_model.py (GPU builder byte for byte against the build model)',
    'link_new_nodes_kernel': 'tests/test_gpu_build_model.py (GPU builder byte for byte against the build model)',
    'reverse_link_kernel': 'tests/test_gpu_build_model.py (GPU builder byte for byte against the build model)',
    'link_new_nodes_cells_kernel': 'tests/test_gpu_build_model.py (one-pass cell-set build against the build model)',
    'reverse_link_cells_kernel': 'tests/test_gpu_build_model.py (one-pass cell-set build against the build model)',
    'filter_eval_kernel<0>': 'tests/test_gpu_attr_filter.py (attribute filters)',
    'filter_eval_kernel<1>': 'tests/test_gpu_attr_filter.py (attribute filters)',
    'rows_copy_kernel': 'tests/test_gpu_attr_filter.py (attribute columns)',
    'filter_compact_kernel': 'tests/test_gpu_attr_filter.py (filter_labels of a prepared filter)',
    'filter_scan_kernel': 'tests/test_gpu_attr_filter.py (filter_labels of a prepared filter)',
    'filter_count_kernel': 'tests/test_gpu_attr_filter.py (filter_labels of a prepared filter)',
    'cell_scatter_kernel': 'tests/test_gpu_cells.py (per-cell parts of the fused cell-set walk)',
    'ivf_merge_kernel': 'tests/test_gpu_cells.py (merged cell-set rows against oracle/ivf.py)',
    'cell_probe_kernel': 'tests/test_gpu_cells.py (GPU probe order against cdist)',
    'subset_count_kernel': 'tests/test_gpu_cells_bruteforce.py (attribute-filter bitmaps scanned exactly)',
    'subset_offsets_kernel': 'tests/test_gpu_cells_bruteforce.py (attribute-filter bitmaps scanned exactly)',
}
