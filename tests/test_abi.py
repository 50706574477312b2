"""The C-ABI library loads and exports every symbol include/geob200.h declares, with matching argument counts
(no compute calls: runs without a GPU)."""
import ctypes
import os
import re

from geotransformer_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_decls():
    hdr = open(os.path.join(ROOT, 'include', 'geob200.h')).read()
    hdr = re.sub(r'/\*.*?\*/', '', hdr, flags=re.S)
    hdr = re.sub(r'typedef struct \{.*?\} \w+;', '', hdr, flags=re.S)
    return re.findall(r'\b(?:int|void|size_t|uint64_t|int64_t|const char\*)\s+(geob200_\w+)\s*\(([^;]*?)\)\s*;', hdr, flags=re.S)


def test_library_exports_every_declared_symbol():
    decls = _header_decls()
    assert len(decls) >= 30
    lib = ctypes.CDLL(L.LIB_PATH)
    for name, args in decls:
        assert hasattr(lib, name), f'{name} declared in geob200.h but not exported'
        n = 0 if args.strip() == 'void' else len(args.split(','))
        assert name in L.SIGNATURES, f'{name} has no ctypes signature'
        assert len(L.SIGNATURES[name][1]) == n, f'{name}: header has {n} args, binding {len(L.SIGNATURES[name][1])}'
    assert set(L.SIGNATURES) == {d[0] for d in decls}


def test_no_torch_types_in_the_abi():
    """signatures use plain pointers and sizes only (comments may cite torch/ATen call sites of the reference)"""
    for name, args in _header_decls():
        for tok in ('at::', 'Tensor', 'torch', 'c10', 'std::'):
            assert tok not in args, f'{name}: {tok} in signature'
    assert 'extern "C"' in open(os.path.join(ROOT, 'include', 'geob200.h')).read()


def test_workspace_queries_work_without_gpu():
    lib = L.lib()
    assert lib.geob200_grid_subsample_workspace_bytes(40000, 2) > 40000 * 40
    assert lib.geob200_radius_search_workspace_bytes(40000, 40000, 2) > 40000 * 20
    assert lib.geob200_lgr_batched_workspace_bytes(1, 256, 64, 3) > 0
    assert lib.geob200_launch_count() == 0


def test_structure_embedding_table_size_and_argument_checks():
    """geob200_gse_table_bytes is pure host arithmetic (header + (nodes_d + nodes_a) x channels x 6 B); the build / embed entry
    points reject bad grids BEFORE any launch (so this runs without a GPU) and leave a message in geob200_last_error()"""
    lib = L.lib()
    nodes = (96 * 256 + 1) + (int(12.25 * 256) + 1)
    assert lib.geob200_gse_table_bytes(256, 256, 96.0, 12.25) == 256 + nodes * 256 * 6
    assert lib.geob200_gse_table_bytes(128, 256, 96.0, 12.25) == 256 + nodes * 128 * 6
    assert lib.geob200_gse_table_bytes(256, 0, 96.0, 12.25) == 0 and lib.geob200_gse_table_bytes(256, 256, -1.0, 12.25) == 0
    buf = ctypes.create_string_buffer(4096)
    bad = [(192, 256, 96.0, 'channels'), (256, 100, 96.0, 'power of two'), (256, 256, 96.0, 'too small')]
    for channels, inv_step, d_max, word in bad:
        rc = lib.geob200_gse_table_build(None, None, None, None, None, channels, inv_step, d_max, 12.25, ctypes.addressof(buf), 4096, None)
        assert rc != 0 and word in lib.geob200_last_error().decode(), (channels, inv_step, lib.geob200_last_error())
    rc = lib.geob200_gse_embed_table(None, None, 10, 256, ctypes.addressof(buf), 4096, 256, 96.0, 12.25, None, None, None, None, None, None, None)
    assert rc != 0 and 'table buffer smaller' in lib.geob200_last_error().decode()
    assert lib.geob200_launch_count() == 0


def test_bad_arguments_are_rejected_before_any_launch():
    """error behaviour of the boundary (the reference raises through TORCH_CHECK, extensions/common/torch_helper.h:6-35): bad sizes /
    empty clouds / non-positive voxel or radius give a negative return code and a message, checked BEFORE any CUDA call -- so this
    runs without a GPU and the launch counter stays at zero"""
    import numpy as np
    lib = L.lib()
    lens = np.array([5, 0], dtype=np.int64)
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)

    def err():
        return lib.geob200_last_error().decode()

    assert lib.geob200_grid_subsample(p, 0, lens.ctypes.data, 2, 0.1, p, p, p, 1 << 16, None) < 0 and 'empty input' in err()
    assert lib.geob200_grid_subsample(p, 5, lens.ctypes.data, 2, 0.0, p, p, p, 1 << 16, None) < 0 and 'voxel' in err()
    assert lib.geob200_grid_subsample(p, 5, lens.ctypes.data, 2, 0.1, p, p, p, 1 << 16, None) < 0 and 'cloud 1 is empty' in err()
    assert lib.geob200_radius_search(p, 0, p, 5, p, p, 1, 0.1, 8, p, p, p, p, 1 << 16, None) < 0 and 'empty input' in err()
    assert lib.geob200_radius_search(p, 5, p, 5, p, p, 1, -1.0, 8, p, p, p, p, 1 << 16, None) < 0 and 'radius' in err()
    assert lib.geob200_neighbor_histogram(p, 0, 8, 5, 16, p, None) < 0 and 'empty input' in err()
    rows = (ctypes.c_int64 * 1)(0)
    assert lib.geob200_gse_indices_batched(p, 1, rows, 0.2, 3.8, 3, p, p, None) < 0 and 'empty cloud' in err()
    rows[0] = 10
    assert lib.geob200_gse_indices_batched(p, 1, rows, 0.2, 3.8, 5, p, p, None) < 0 and 'angle_k' in err()
    assert lib.geob200_launch_count() == 0


def test_product_does_not_import_the_oracle():
    """the oracle is test infrastructure: nothing under geotransformer_b200/ may reference it"""
    pkg = os.path.join(ROOT, 'geotransformer_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                src = open(os.path.join(dirpath, f)).read()
                assert 'import oracle' not in src and 'from oracle' not in src and 'liboracle' not in src and 'libref_ext' not in src, f
