"""The compact wire format of csrc/batch_wire.cu (chg_pack_batch_wire) against the full format (chg_pack_batch_host):
every field of the batch descriptor must come out identical, and graphs that break the format's assumptions must be
detected while packing and shipped in full (reference semantics: BatchedGraph.from_graphs, model.py:792-913, uses every
column as given)."""
import copy
import dataclasses

import dense_cells
import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch


def _assert_same(a, b):
    n = 0
    for f in dataclasses.fields(a):
        x, y = getattr(a, f.name), getattr(b, f.name)
        if isinstance(x, torch.Tensor):
            assert x.dtype == y.dtype and x.shape == y.shape, f.name
            assert torch.equal(x, y), f.name
            n += 1
        elif f.name != "h2d_bytes":
            assert x == y, f.name
    assert n >= 30


def _cases():
    g_far = graphgen.make_crystal_graph([3, 8], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.eye(3) * 5.5)
    g_iso = graphgen.make_crystal_graph([1, 1], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.eye(3) * 20.0)
    g_thin = graphgen.make_crystal_graph([3, 8], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.diag([2.2, 2.4, 9.0]))  # images up to +-3
    z, frac, lat = graphgen.limno2_structure((3, 2, 2), 0.02, 4001)
    big = graphgen.make_crystal_graph(z, frac, lat)
    return [graphgen.random_graphs(5, 8, 30, 9100), [g_iso], [g_far], [g_thin], [g_iso, g_far, g_thin] + graphgen.random_graphs(2, 9, 12, 9200),
            graphgen.random_graphs(40, 10, 30, 1000), [big], dense_cells.dense_graphs()]


@pytest.mark.parametrize("case", range(8))
def test_wire_format_equals_full_format_cpu(case):
    graphs = _cases()[case]
    _assert_same(build_batch(graphs, "cpu", wire=True), build_batch(graphs, "cpu", wire=False))


def test_wire_format_threads_split_one_large_graph(monkeypatch):
    """A single graph above the threading threshold is packed in slices by several workers."""
    z, frac, lat = graphgen.limno2_structure((5, 4, 4), 0.02, 11)
    g = graphgen.make_crystal_graph(z, frac, lat)
    assert g.atom_graph.shape[0] * 6 + g.bond_graph.shape[0] * 5 > (1 << 18)
    _assert_same(build_batch([g], "cpu", wire=True), build_batch([g], "cpu", wire=False))


def _lib_flags(graphs):
    import ctypes

    from chgnet_b200 import batch as B

    infos = [g.pack_info() for g in graphs]
    counts = np.ascontiguousarray(np.stack([i[0] for i in infos]))
    ptrs = np.ascontiguousarray(np.stack([i[1] for i in infos]))
    n, ed, eu, an = (int(v) for v in counts.sum(0))
    ib = torch.empty(2 * n + 3 * ed + eu + 2 * an + 1, dtype=torch.int32)
    fb = torch.empty(3 * n + 9 * len(graphs), dtype=torch.float32)
    im = torch.empty(3 * ed + 1, dtype=torch.int8)
    flags = (ctypes.c_int32 * 5)()
    rc = B._pack_lib().chg_pack_batch_wire(len(graphs), counts.ctypes.data, ptrs.ctypes.data, ib.data_ptr(), fb.data_ptr(),
                                           im.data_ptr(), None, None, None, flags, None)
    assert rc == 0
    return list(flags)


def test_graphs_outside_the_format_are_detected_and_shipped_in_full():
    base = graphgen.random_graphs(3, 10, 14, 77)
    assert _lib_flags(base)[4] == 0
    g = base[1]
    # (1) a bond-graph column that is NOT the function of the directed-edge columns the format assumes
    bad = copy.copy(g)
    bg = g.bond_graph.clone()
    bg[0, 1] = (bg[0, 1] + 1) % g.undirected2directed.shape[0]
    bad.bond_graph = bg
    assert _lib_flags([base[0], bad])[4] == 2
    _assert_same(build_batch([base[0], bad], "cpu", wire=True), build_batch([base[0], bad], "cpu", wire=False))
    # (2) an image that does not fit int8, (3) a fractional image
    for val in (300.0, 0.5):
        wide = copy.copy(g)
        im = g.neighbor_image.clone()
        im[2, 1] = val
        wide.neighbor_image = im
        assert _lib_flags([wide])[4] == 1
        _assert_same(build_batch([wide], "cpu", wire=True), build_batch([wide], "cpu", wire=False))
    # (4) a directed-edge index outside the graph
    oob = copy.copy(g)
    bg = g.bond_graph.clone()
    bg[1, 4] = g.atom_graph.shape[0] + 5
    oob.bond_graph = bg
    assert _lib_flags([oob])[4] == 3


def test_wire_format_reports_bad_atomic_number():
    g = copy.copy(graphgen.random_graphs(1, 10, 12, 5)[0])
    zt = g.atomic_number.clone()
    zt[3] = 95
    g.atomic_number = zt
    with pytest.raises(IndexError, match="atomic number 95"):
        build_batch([g], "cpu", wire=True)


@pytest.mark.gpu
def test_wire_format_equals_full_format_gpu():
    """Same comparison through the device path: copies in two phases + expand_image / derive_angle_columns kernels."""
    for graphs in _cases() + [graphgen.random_graphs(64, 40, 60, 1000)]:
        for with_reverse in (True, False):
            a = build_batch(graphs, "cuda", with_reverse=with_reverse, wire=True)
            b = build_batch(graphs, "cuda", with_reverse=with_reverse, wire=False)
            _assert_same(a, b)
            assert a.h2d_bytes < b.h2d_bytes or a.n_edges == 0
    # repeated calls reuse the pinned staging buffers while earlier copies may still be in flight
    graphs = graphgen.random_graphs(32, 20, 40, 3)
    ref = build_batch(graphs, "cuda", wire=False)
    outs = [build_batch(graphs, "cuda", wire=True) for _ in range(5)]
    torch.cuda.synchronize()
    for o in outs:
        _assert_same(o, ref)


def test_packer_is_safe_under_concurrent_callers():
    """Two Python threads batching different graph lists at the same time: the library's worker pool runs one job at a
    time (worker_pool.h), so both get exactly what a single caller gets.  (Staging buffers are per process: the CPU
    'device' clones out of them before returning, like the device path copies out of them.)"""
    import threading

    # above the threading threshold, so the workers are actually used
    sets = [graphgen.random_graphs(48, 20, 40, 500 + k) for k in range(2)]
    want = [build_batch(s, "cpu", wire=False) for s in sets]
    errors = []
    lock = threading.Lock()

    def work(k):
        try:
            for _ in range(4):
                with lock:  # build_batch itself reuses per-process staging buffers: one Python caller at a time
                    got = build_batch(sets[k], "cpu", wire=True)
                _assert_same(got, want[k])
        except Exception as exc:  # noqa: BLE001
            errors.append(repr(exc))

    threads = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors
    # and the raw C entry point from two threads at once, each with its own buffers
    from chgnet_b200 import batch as B
    import ctypes

    def raw(k, out):
        infos = [g.pack_info() for g in sets[k]]
        counts = np.ascontiguousarray(np.stack([i[0] for i in infos]))
        ptrs = np.ascontiguousarray(np.stack([i[1] for i in infos]))
        n, ed, eu, an = (int(v) for v in counts.sum(0))
        ib = torch.empty(2 * n + 3 * ed + eu + 2 * an + 1, dtype=torch.int32)
        fb = torch.empty(3 * n + 9 * len(infos), dtype=torch.float32)
        im = torch.empty(3 * ed + 1, dtype=torch.int8)
        flags = (ctypes.c_int32 * 5)()
        for _ in range(6):
            rc = B._pack_lib().chg_pack_batch_wire(len(infos), counts.ctypes.data, ptrs.ctypes.data, ib.data_ptr(), fb.data_ptr(),
                                                   im.data_ptr(), None, None, None, flags, None)
            assert rc == 0 and flags[4] == 0
        out[k] = (ib[2 * n: 2 * n + ed].clone(), n, ed)

    out = {}
    threads = [threading.Thread(target=raw, args=(k, out)) for k in range(2)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    for k in range(2):
        center, n, ed = out[k]
        assert torch.equal(center, want[k].center)
