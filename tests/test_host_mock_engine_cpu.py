"""CPU: libmkhost's engine-facing packers run against the CPU mock of libmksnap (tests/mock_engine/mock_mksnap.cpp:
every digest computed by the oracle, the same call contract enforced).  Each scenario runs in a fresh process that
loads the mock with RTLD_GLOBAL before libmkhost, so the real host code -- arena flushing, stream continuation, ranges
per file, untar / materialise from the arena -- executes exactly as it does on an H100, minus the kernels.  These are
the CPU twins of tests/test_gpu_host.py and tests/test_gpu_host_arena_paths.py."""
import os

import pytest

from tests import mock_engine


@pytest.mark.skipif(os.geteuid() != 0, reason="chown needs root")
@pytest.mark.parametrize("scenario", ["cache_id_and_commit", "ingest_untar_and_file_digests", "content_aware_scan",
                                      "materialize_from_the_arena", "random_trees_small_arenas",
                                      "table_limits_and_arena_leases", "batch_of_layers_in_one_session",
                                      "ingest_member_larger_than_the_arena", "incremental_cache_id"])
def test_host_packers_against_the_mock_engine(tmp_path, scenario):
    r = mock_engine.run("tests.mock_engine.run", scenario, tmp_path)
    assert "SCENARIO-OK" in r.stdout, r.stdout[-3000:]
