"""GPU: kernels of libmgb200.so (CUDA, sm_90a) on their own, launched as the mapping pipeline launches them -- the on-chip WFA
tiers, the bridging alignment and the exact radix sort of the seeds -- against the reference functions they restate."""
import pytest

import cases
import mgtest as T
from minigraph_b200 import capi

pytestmark = pytest.mark.gpu

# shared memory k_seed gives the seed sort (mgb_seed.cuh SKETCH_SMEM_BYTES)
SEED_SORT_SMEM = 12 * 32 * 16


@pytest.fixture(scope="module")
def lib():
    return capi.load_product()


@pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not shipped")
@pytest.mark.parametrize("tier", [1, 2])
def test_wfa_tier_limits(lib, tier):
    cases.case_wfa_tier_edges(lib, tier, scale=2)


def test_wfa_tier_refuses_empty_sides(lib):
    cases.case_wfa_tier_rejects_empty(lib)


@pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not shipped")
def test_bridging_alignment(lib, workdir):
    cases.case_gwfa_bridges(lib, workdir, scale=4)


def test_bridging_refuses_bad_input(lib, workdir):
    cases.case_gwfa_rejects_bad_input(lib, workdir)


def test_exact_radix_sort(lib):
    cases.case_radix_exact(lib, hot_max=SEED_SORT_SMEM)
