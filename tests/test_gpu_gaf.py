"""mgb_map_batch_gaf() on the GPU: GAF text formatted by the device kernels (k_gaf_count / k_gaf_write), byte for byte against the
reference's golden files and the host writer."""
import pytest

import gafcases as GC
from minigraph_b200 import capi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return capi.load_product()


def test_existing_goldens(lib, workdir):
    GC.case_existing_goldens(lib, workdir)


def test_output_option_goldens_and_host_writer(lib, workdir):
    GC.case_flag_goldens(lib, workdir)


def test_read_pairs(lib, workdir):
    GC.case_pairs(lib, workdir)


def test_empty_batch_null_names_buffer_reuse_refusals(lib, workdir):
    GC.case_api(lib, workdir)


def test_config2_full_size(lib, workdir):
    GC.case_full_c2(lib, workdir)


def test_concurrent_callers(lib, workdir):
    GC.case_concurrent(lib, workdir)


def test_several_devices(lib, workdir):
    GC.case_multi_device(lib, workdir)


def test_without_label_cache(lib, workdir):
    GC.case_no_label_cache(lib, workdir)
