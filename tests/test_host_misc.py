"""CPU: small host-side pieces -- enums, argument validation of the Python surface, bench helpers,
and the SASS evidence that the shipped library is an sm_90a build that uses TMA bulk copies."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT


def test_metric_enum_matches_reference_names():
    from annlite_b200 import ExpandMode, Metric
    assert [m.name for m in Metric] == ['EUCLIDEAN', 'INNER_PRODUCT', 'COSINE'] and Metric.COSINE == 3
    assert Metric.from_string('cosine') is Metric.COSINE and str(Metric.EUCLIDEAN) == 'EUCLIDEAN'
    with pytest.raises(ValueError):
        Metric.from_string('manhattan')
    assert ExpandMode.STEP == 1


def test_annlite_rejects_out_of_scope_configurations(tmp_path):
    from annlite_b200 import AnnLite
    with pytest.raises(NotImplementedError, match='n_cells'):
        AnnLite(32, n_cells=4, n_subvectors=4, data_path=tmp_path)
    with pytest.raises(NotImplementedError, match='PCA'):
        AnnLite(32, n_components=8, n_subvectors=4, data_path=tmp_path)
    with pytest.raises(NotImplementedError, match='n_subvectors'):
        AnnLite(32, data_path=tmp_path)
    with pytest.raises(AssertionError):
        AnnLite(30, n_subvectors=4, data_path=tmp_path)


def test_host_math_matches_reference_definitions():
    from annlite_b200.math import l2_normalize, top_k
    rng = np.random.default_rng(0)
    x = rng.standard_normal((5, 7)).astype(np.float32)
    x[2] = 0
    n = l2_normalize(x)
    assert np.allclose(np.linalg.norm(n[[0, 1, 3, 4]], axis=1), 1, atol=1e-6) and (n[2] == 0).all()
    v = rng.random((3, 50))
    d, i = top_k(v, 5)
    assert np.array_equal(i, np.argsort(v, axis=1)[:, :5]) and np.array_equal(d, np.sort(v, axis=1)[:, :5])
    d, i = top_k(v, 80)
    assert i.shape == (3, 50)


def test_hnsw_bind_index_needs_pq():
    from annlite_b200.hnsw_bind import Index
    with pytest.raises(RuntimeError, match='Space name'):
        Index(space='hamming', dim=8)
    idx = Index(space='l2', dim=8)
    idx.init_index(max_elements=10)
    assert idx.index_inited and not idx.pq_enable and idx.element_count == 0
    with pytest.raises(NotImplementedError, match='PQ-encoded'):
        idx.knn_query(np.zeros((1, 8), np.float32), k=1, dtables=np.zeros((1, 2, 4), np.float32))
    with pytest.raises(RuntimeError, match='already initiated'):
        idx.init_index(max_elements=10)

    class Bad:
        pass
    with pytest.raises(IndexError, match='PQ class should at least'):
        Index(space='l2', dim=8).init_index(10, pq_codec=Bad())


def test_bench_synthetic_data_is_reproducible_by_slice():
    sys.argv = ['bench.py', '--n', '250000']
    sys.path.insert(0, ROOT)
    import bench
    a = bench.parse()
    full = bench.make_base(a, 90_000, 210_000)
    assert np.array_equal(full[20_000:30_000], bench.make_base(a, 110_000, 120_000))
    assert bench.cfg_key(a) != bench.cfg_key(a, 'shard0of2')
    q0, q1 = bench.make_queries(a, 2, rank=0), bench.make_queries(a, 2, rank=1)
    assert q0.shape == (2, a.batch, a.dim) and not np.array_equal(q0, q1)


def test_shipped_library_is_an_sm90a_build_with_tma():
    from annlite_b200 import _lib
    lst = subprocess.run(['cuobjdump', '-lelf', _lib.LIB_PATH], capture_output=True, text=True)
    if lst.returncode != 0:
        pytest.skip('cuobjdump unavailable')
    assert 'sm_90a' in lst.stdout and 'sm_100' not in lst.stdout and 'sm_80' not in lst.stdout
    sass = subprocess.run(['cuobjdump', '-sass', _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert 'UBLKCP' in sass            # cp.async.bulk: the per-query table is staged by TMA
    assert 'SYNCS.ARRIVE.TRANS64' in sass   # mbarrier expect_tx
    assert 'HMMA' not in sass and 'HGMMA' not in sass   # no tensor-core path on this (gather-bound) workload


def test_committed_bench_line_follows_the_contract():
    """The JSON line bench.py printed on an H100 (profiles/h100_bench_n1.json) carries every key the
    measurement contract asks for."""
    import json
    d = json.loads(open(os.path.join(ROOT, 'profiles', 'h100_bench_n1.json')).read().strip().splitlines()[-1])
    for key in ['metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling',
                'vs_baseline', 'dtype', 'data', 'config', 'e2e', 'gpu_launches', 'clocks', 'roofline', 'cpu_baseline', 'parity']:
        assert key in d, key
    assert d['higher_is_better'] is True and d['vs_baseline'] is None and d['data'] == 'synthetic' and d['dtype'] == 'f32'
    assert 'workload' in d['config'] and 'model' not in d['config']
    r = d['roofline']
    assert r['bound'] == 'hbm' and abs(r['frac'] - r['achieved'] / r['peak']) < 1e-3
    e = d['e2e']
    assert e['h2d_bytes_per_step'] == 10_000 * 128 * 4 and e['d2h_bytes_per_step'] > 0 and e['value'] != d['value']
    c = d['cpu_baseline']
    assert c['kind'] in ('port', 'reference') and c['cores'] >= 1 and 'sample' in c
    assert d['gpu_launches'] == d['steps']                # ONE kernel per step: the table build is inside the walk
    # no hardware or thermal slowdown; the card's own power cap may engage, but then its limit is stated beside the number
    # and the clocks held
    assert set(d['clocks']['reasons']) <= {'sw_power_cap'} and d['clocks']['sm_mhz'] >= 0.9 * d['clocks']['sm_max_mhz']
    assert 'H100' in d['gpu']['name'] and d['gpu']['power_limit_w'] > 0 and d['gpu']['sms'] == 132
    p = d['parity']
    assert p['rows'] == 10_000 and p['diff'] <= 2 and p['exact'] + p['tie'] + p['diff'] == p['rows']
    ref = json.loads(open(os.path.join(ROOT, 'profiles', 'h100_bench_reference.json')).read().strip().splitlines()[-1])
    assert ref['impl'] == 'reference' and ref['cpu_baseline']['kind'] == 'reference' and ref['e2e']['h2d_bytes_per_step'] == 0
    assert ref['metric'] == d['metric'] and ref['unit'] == d['unit'] and 'recall_at_k' in ref
