"""decode_sequential_kernel -- the one-thread-per-chunk parser of raw / XOR / Gorilla streams -- on the plans that the
parallel boundary searches (decode_mixed_kernel, decode_gorilla_kernel) take by default. The sequential parser stays
because overlapping fields and two or more Gorilla fields need it; CLDN_B200_MIXED_DECODE=seq sends every such plan to
it. Every test here re-runs a parity test of test_gpu_parity.py / test_gpu_ros.py with that switch set.
It sorts last on purpose (a surprise here cannot hide the defaults' results behind `pytest -x`)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_parity as P  # noqa: E402
import test_gpu_ros as R  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _legacy_kernels(monkeypatch):
    monkeypatch.setenv("CLDN_B200_MIXED_DECODE", "seq")


def test_golden_vectors(golden, oracle):            # v2 goldens: XOR / Gorilla coders of the reference, wire versions 3 / 4 / 5
    P.test_golden_vectors(golden, oracle)


@pytest.mark.parametrize("version", [5, 4, 3])
@pytest.mark.parametrize("lossless", [True, False])
def test_lossless_float_fields(oracle, version, lossless):
    P.test_lossless_float_fields(oracle, version, lossless)


@pytest.mark.parametrize("mode", ["seq"])
@pytest.mark.parametrize("version", [5, 4])
def test_raw_fields_in_the_stream(oracle, monkeypatch, mode, version):
    P.test_raw_fields_in_the_stream(oracle, monkeypatch, mode, version)


def test_gorilla_field_positions(oracle, monkeypatch):
    P.test_gorilla_field_positions(oracle, monkeypatch, "seq")


def test_v5_section_decode_errors():
    P.test_v5_section_decode_errors()


def test_skip_store(oracle, monkeypatch):
    P.test_decode_but_skip_store(oracle, monkeypatch, "seq")
    P.test_skip_store_in_v5_sections_is_honoured_here()


def test_c4_velodyne_mixed_layout(oracle):
    P.test_c4_velodyne_mixed_layout(oracle)


def test_corrupted_blobs_decode_like_the_reference(ref):
    P.test_corrupted_blobs_decode_like_the_reference(ref)


def test_dds_paths(ref, golden_ros):                 # the reference's sample layout (FLOAT64 timestamp -> Gorilla) through the envelope
    R.test_dds_roundtrip_like_the_reference_test(golden_ros)
    R.test_compress_message_matches_reference(ref, False)
    R.test_decompress_message_matches_reference(ref)
    R.test_golden_messages(golden_ros)


def test_reference_sample_files(oracle):             # only where the reference tree exists (tests/cusim)
    P.test_reference_sample_files(oracle)
