"""mgb_map_batch_gaf() in both simulators of the device code (one lane, and 32 lanes as fibres, which run the warp scans and the
lane-parallel CIGAR / ds:Z / delta writes the GPU runs): GAF text byte for byte against the reference's golden files, and against
the host writer over mg_map_batch() results under every GAF output option; a batch split over several devices (MGB_DEVICES) gives
the text of one."""
import pytest

import gafcases as GC
import mgtest as T


@pytest.fixture(scope="module", params=["hostsim", "hostsim32"])
def lib(request):
    return T.load_hostsim() if request.param == "hostsim" else T.load_hostsim32()


def test_existing_goldens(lib, workdir):
    GC.case_existing_goldens(lib, workdir)


def test_output_option_goldens_and_host_writer(lib, workdir):
    GC.case_flag_goldens(lib, workdir)


def test_read_pairs(lib, workdir):
    GC.case_pairs(lib, workdir)


def test_goldens_reach_the_traps():
    GC.case_goldens_reach_the_traps()


def test_empty_batch_null_names_buffer_reuse_refusals(lib, workdir):
    GC.case_api(lib, workdir)


def test_several_devices(lib, workdir):
    GC.case_multi_device(lib, workdir)


@pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built")
def test_random_graphs_vs_reference(lib, workdir):
    GC.case_random_vs_reference(lib, workdir)
