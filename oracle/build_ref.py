#!/usr/bin/env python
"""Build the *real* reference native path into ``oracle/_ref/`` (TEST INFRASTRUCTURE ONLY).

What it does
------------
Compiles the reference's two native extensions from the sources where they lie under
``/root/reference`` -- nothing is copied into this repository, only the two built ``.so``
files land in ``oracle/_ref/`` (git-ignored, but shipped to the GPU box by ``gpurun``):

* ``pq_bind``   <- ``bindings/pq_bindings.pyx``        (Cython, C++ mode; setup.py:51-55)
* ``hnsw_bind`` <- ``bindings/hnsw_bindings.cpp`` + ``include/hnswlib/*.h`` (pybind11)

Flags follow ``setup.py:125-151`` (``-O3 -fopenmp -std=c++14`` => ISO mode => no FMA
contraction) except ``-march=native`` -> ``-march=x86-64-v3``: the artefact is built in a
CPU-only container and executed on a different host (the GPU host); the PQ path is scalar
table look-ups, so the ISA level only guards against SIGILL, it does not change results.

One build-time edit is applied to a *temporary* copy of ``hnsw_bindings.cpp``
(SURVEY.md section 0.4): ``knnQuery_return_numpy_`` constructs a ``py::array_t`` after
``py::gil_scoped_release`` (hnsw_bindings.cpp:312-326), which segfaults on
Python 3.12 / pybind11 3.x.  The release statement is moved below the ``dtables`` block,
exactly where ``knnQuery_with_filter_`` already has it (hnsw_bindings.cpp:411-451).  No
semantic change; ``knn_query_with_filter(filters=all ids)`` on the unpatched file returns
identical results (checked in tests/test_oracle_vs_ref.py when /root/reference exists).

Usage: ``python oracle/build_ref.py [--ref /root/reference] [--force]``
"""
import argparse
import os
import shutil
import subprocess
import sys
import sysconfig
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, '_ref')

CXXFLAGS = ['-O3', '-march=x86-64-v3', '-fopenmp', '-std=c++14', '-fPIC', '-shared',
            '-fvisibility=hidden', '-w']


def _ext_suffix():
    return sysconfig.get_config_var('EXT_SUFFIX') or '.so'


def _py_includes():
    import numpy
    import pybind11
    return ['-I' + sysconfig.get_paths()['include'], '-I' + numpy.get_include(),
            '-I' + pybind11.get_include()]


def _hoist_gil_release(src: str) -> str:
    """Move the GIL release in knnQuery_return_numpy_ below the dtables block."""
    lines = src.split('\n')
    start = next(i for i, l in enumerate(lines) if 'knnQuery_return_numpy_(size_t k' in l)
    rel = next(i for i in range(start, len(lines)) if 'py::gil_scoped_release' in lines[i])
    dst = next(i for i in range(rel, len(lines)) if 'if (num_threads <= 0)' in lines[i])
    release_line = lines.pop(rel)
    lines.insert(dst - 1, release_line)
    return '\n'.join(lines)


def build(ref='/root/reference', force=False, verbose=True):
    suffix = _ext_suffix()
    targets = [os.path.join(OUT, 'pq_bind' + suffix), os.path.join(OUT, 'hnsw_bind' + suffix)]
    if not force and all(os.path.exists(t) for t in targets):
        return targets
    if not os.path.isdir(ref):
        raise FileNotFoundError(f'reference tree {ref} not present; cannot (re)build oracle/_ref')
    os.makedirs(OUT, exist_ok=True)
    inc = _py_includes()
    with tempfile.TemporaryDirectory(prefix='annb_ref_') as tmp:
        # --- pq_bind (Cython -> C++) -------------------------------------------------
        pyx = os.path.join(tmp, 'pq_bind.pyx')
        shutil.copy(os.path.join(ref, 'bindings', 'pq_bindings.pyx'), pyx)
        cpp = os.path.join(tmp, 'pq_bind.cpp')
        subprocess.check_call([sys.executable, '-m', 'cython', '--cplus', '-3',
                               '--module-name', 'pq_bind', pyx, '-o', cpp])
        subprocess.check_call(['g++', *CXXFLAGS, *inc, cpp, '-o', targets[0]])
        # --- hnsw_bind (pybind11) ----------------------------------------------------
        with open(os.path.join(ref, 'bindings', 'hnsw_bindings.cpp')) as f:
            src = _hoist_gil_release(f.read())
        hcpp = os.path.join(tmp, 'hnsw_bind.cpp')
        with open(hcpp, 'w') as f:
            f.write(src)
        subprocess.check_call(['g++', *CXXFLAGS, *inc,
                               '-I' + os.path.join(ref, 'include', 'hnswlib'),
                               hcpp, '-o', targets[1], '-pthread'])
    if verbose:
        print('built', *targets, sep='\n  ')
    return targets


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--ref', default='/root/reference')
    ap.add_argument('--force', action='store_true')
    a = ap.parse_args()
    build(a.ref, a.force)
