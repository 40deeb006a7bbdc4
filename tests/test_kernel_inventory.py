"""Every kernel entry of the built library is accounted for (CPU): checked by a GPU case of tests/test_gpu_instances.py
or run by a named test of another path.  A new template instantiation nobody checks, or a case that claims a kernel
the library does not contain, fails here."""
import re

import pytest

import kernel_cases as K


@pytest.fixture(scope='module')
def keys():
    from annlite_b200 import _lib
    if K._tool('cuobjdump') is None or K._tool('cu++filt') is None:
        pytest.skip('cuobjdump / cu++filt not found')
    return K.library_keys(_lib.LIB_PATH)


@pytest.mark.parametrize('name,key', [
    ('void <unnamed>::hnsw_walk4<(int)16, (int)16, (bool)0>(GraphDev, SearchParams)', 'hnsw_walk4<16,16,0>'),
    ('void (anonymous namespace)::hnsw_walk4<16, 16, false>(GraphDev, SearchParams)', 'hnsw_walk4<16,16,0>'),
    ('void (anonymous namespace)::hnsw_walk4f<8, 2, 3, true, (bool)1>(GraphDev, SearchParams, int)', 'hnsw_walk4f<8,2,3,1,1>'),
    ('void <unnamed>::scan_topk_kernel<(int)2, unsigned short>(const float *, const T2 *, long)', 'scan_topk_kernel<2,u16>'),
    ('void <unnamed>::merge_topk_kernel<unsigned int, long, (int)1>(const float *, T2 *, T1, T2)', 'merge_topk_kernel<u32,i64,1>'),
    ('merge_sorted_kernel(const float *, const unsigned long *, int, long, int, long, long, float *, unsigned long *)', 'merge_sorted_kernel'),
    ('<unnamed>::reverse_link_cells_kernel(const <unnamed>::BuildDev *, const int *)', 'reverse_link_cells_kernel'),
    ('void <unnamed>::filter_eval_kernel<(bool)1>(const annb_filter_op_t *, int)', 'filter_eval_kernel<1>'),
    ('void <unnamed>::encode_kernel<unsigned char>(const float *, const float *, T1 *, long, int, int, int)', 'encode_kernel<u8>'),
])
def test_kernel_key_normalises_both_name_forms(name, key):
    assert K.kernel_key(name) == key


def test_the_two_groups_are_disjoint():
    assert not (K.COVERED & set(K.ELSEWHERE))
    assert all(re.search(r'tests/test_\w+\.py', t) for t in K.ELSEWHERE.values())


def test_every_library_kernel_is_covered_or_run_elsewhere(keys):
    assert len(keys) > 380
    unaccounted = keys - K.COVERED - set(K.ELSEWHERE)
    assert not unaccounted, sorted(unaccounted)


def test_every_kernel_a_case_claims_is_in_the_library(keys):
    phantom = (K.COVERED | set(K.ELSEWHERE)) - keys
    assert not phantom, sorted(phantom)


def test_every_named_test_exists():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for key, where in K.ELSEWHERE.items():
        path = re.search(r'tests/test_\w+\.py', where).group(0)
        assert os.path.exists(os.path.join(root, path)), (key, path)
