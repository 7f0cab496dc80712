"""-m gpu: the sharded layer ingest of libmkhost (mkhost_memfs_update_from_tars_multi) on libmksnap.  The scenarios of
tests/mock_engine/multi_ingest_cases.py -- each compares 1, 2, 3 and 5 engines with update_from_tars_cached on one
engine -- with every engine on device 0 and arenas of 1 MiB, so each engine submits several times; then a cold and a
warm run with one engine per device (skipped with fewer than two)."""
import pytest

from tests.mock_engine import multi_ingest_cases as cases
from tests.test_gpu_multi_engine import make_engine

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scenario", cases.ALL)
def test_multi_ingest_one_device(scenario, tmp_path):
    getattr(cases, scenario)(make_engine, str(tmp_path))


def test_multi_ingest_one_engine_per_device(tmp_path):
    import torch
    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("needs two or more GPUs")
    from makisu_b200 import host
    k = [0]

    def make(arena, **kw):  # round robin over the devices
        k[0] += 1
        return make_engine(arena, device=(k[0] - 1) % n_dev, **kw)

    layers = cases.lcc.layer_set()
    paths, keys, run = cases._setup(str(tmp_path), layers)
    run.make = make
    lc, gz = host.LayerCache(), host.GzIndexCache()
    for _ in range(2):  # cold, then warm: every layer replayed on engine 0
        k[0] = 0
        cases.check(run, make, n_dev, paths, layers, keys, host.MKHOST_FILE_DIGESTS, lc, gz)
