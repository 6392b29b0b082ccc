import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (run with -m gpu)")


# Collection order: the cheapest, most local checks first, so that a `-x` run stops at the real culprit (a broken kernel fails its
# own known-answer test before it fails a whole-scene trajectory).  Within one rank the file / definition order is kept.
_ORDER = [
    "test_host", "test_oracle_kat", "test_transfer_kat", "test_stage_kat", "test_variants_emulated", "test_slab_gloo", "test_bench_contract",
    "test_gpu_pcg", "test_gpu_transfer", "test_gpu_parity", "test_golden", "test_gpu_solids", "test_zz_mesh_voxelizer", "test_gpu_runner",
    "test_gpu_configs", "test_gpu_fullsize", "test_gpu_multi",
]


def pytest_collection_modifyitems(session, config, items):
    def rank(item):
        name = os.path.splitext(os.path.basename(str(item.fspath)))[0]
        return _ORDER.index(name) if name in _ORDER else len(_ORDER)

    items.sort(key=rank)  # stable
