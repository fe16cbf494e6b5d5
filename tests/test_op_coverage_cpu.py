"""Coverage ledger of the C ABI: every entry point declared in include/b200sep.h is called by name (`lib.<symbol>(...)`) in at least one GPU
test (tests/test_*_gpu.py), or is listed in INDIRECT with the reason it is not.  A mention in a comment or a string does not count.  A new
entry point without a test fails here, on the CPU."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# symbol -> why no GPU test names it
INDIRECT = {
    # queries, handles and measurement hooks: no numeric result of their own
    "b200sep_abi_version": "checked when _lib.py loads the library (every test imports it)",
    "b200sep_launch_count": "launch counter read by bench.py through _lib.launch_count()",
    "b200sep_stft_plan_destroy": "destructor",
    "b200sep_mdxnet_destroy": "destructor",
    "b200sep_tfcnet_destroy": "destructor",
    "b200sep_graph_destroy": "destructor",
    "b200sep_mdxnet_param_count": "size query used by engine.MdxNet when it packs the weights",
    "b200sep_mdxnet_device_bytes": "size query",
    "b200sep_tfcnet_param_count": "size query used by engine.TfcNet; test_abi_and_host.py checks it against the reference state_dict",
    "b200sep_tfcnet_device_bytes": "size query",
    "b200sep_flac_work_bytes": "size query of the FLAC encoder's scratch",
    "b200sep_flac_max_bytes": "size query of the FLAC encoder's output bound",
    "b200sep_flac_decode_work_bytes": "size query of the FLAC decoder's scratch",
    "b200sep_mdxnet_profile_enable": "measurement hook of bench.py's roofline",
    "b200sep_mdxnet_profile_read": "measurement hook of bench.py's roofline",
    "b200sep_mdxnet_profile_name": "measurement hook of bench.py's roofline",
    "b200sep_capture_begin": "CUDA-graph capture of the engines' launch lists (graphs.py); the separation goldens run through it",
    "b200sep_capture_end": "CUDA-graph capture of the engines' launch lists (graphs.py); the separation goldens run through it",
    "b200sep_graph_launch": "CUDA-graph capture of the engines' launch lists (graphs.py); the separation goldens run through it",
    # whole operators called through their Python wrappers, each with its own operator-level test against an oracle
    "b200sep_stft_plan_create": "engine.StftPlan; test_mdx_gpu.py::test_stft_forward_inverse_vs_oracle",
    "b200sep_stft_forward": "engine.StftPlan; test_mdx_gpu.py::test_stft_forward_inverse_vs_oracle and test_stft_vs_reference_golden",
    "b200sep_stft_inverse": "engine.StftPlan; test_mdx_gpu.py::test_stft_forward_inverse_vs_oracle and test_stft_vs_reference_golden",
    "b200sep_mdxnet_create": "engine.MdxNet; test_mdx_gpu.py::test_network_small_vs_oracle_and_golden",
    "b200sep_mdxnet_forward": "engine.MdxNet; test_mdx_gpu.py::test_network_small_vs_oracle_and_golden and test_network_full_size_chunk_vs_golden",
    "b200sep_tfcnet_create": "engine.TfcNet; test_mdxc_gpu.py::test_tfcnet_spec_vs_reference_golden",
    "b200sep_tfcnet_forward": "engine.TfcNet; test_mdxc_gpu.py::test_tfcnet_spec_vs_reference_golden",
    "b200sep_resample_sinc_f32": "b200/resample.py; test_resample_gpu.py::test_kernel_vs_oracle_ratios and _five_minutes against oracle/resample_oracle.py",
    "b200sep_flac_encode": "b200/flac.py; test_flac_gpu.py::test_lossless_roundtrip_matrix (bit-exact against the CPU decoder oracle)",
    "b200sep_flac_locate": "b200/flac.py; test_flac_decode_gpu.py::test_writer_streams and test_damaged_streams against the stream oracle",
    "b200sep_flac_decode": "b200/flac.py; test_flac_decode_gpu.py::test_writer_streams and test_damaged_streams against the stream oracle",
}


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "b200sep.h")).read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"//[^\n]*", " ", text)
    return sorted(set(re.findall(r"\b(b200sep_\w+)\s*\(", text)))


def called(sym, text):
    """a call through the ctypes handle, e.g. lib.b200sep_x( or L.lib.b200sep_x("""
    return re.search(r"\.%s\s*\(" % sym, text) is not None


def gpu_test_texts():
    return {os.path.basename(f): open(f).read() for f in sorted(glob.glob(os.path.join(ROOT, "tests", "test_*_gpu.py")))}


def test_header_parses():
    syms = declared_symbols()
    assert len(syms) > 100
    assert "b200sep_groupnorm1_f32" in syms and "b200sep_graph_destroy" in syms
    assert not any(s.startswith("b200sep_stft_plan") and not s.endswith(("_create", "_destroy")) for s in syms)
    assert called("b200sep_absmax", "check(L.lib.b200sep_absmax (x))") and not called("b200sep_absmax", "# see b200sep_absmax(...)")


def test_every_entry_point_is_tested_or_listed():
    texts = gpu_test_texts()
    untested = [s for s in declared_symbols() if s not in INDIRECT and not any(called(s, t) for t in texts.values())]
    assert not untested, f"entry points no tests/test_*_gpu.py calls by name (add a test, or list them in INDIRECT with a reason): {untested}"


def test_indirect_table_is_current():
    syms = set(declared_symbols())
    stale = sorted(set(INDIRECT) - syms)
    assert not stale, f"INDIRECT lists symbols the header no longer declares: {stale}"
    texts = gpu_test_texts()
    named = sorted(s for s in INDIRECT if any(called(s, t) for t in texts.values()))
    assert not named, f"INDIRECT lists symbols a GPU test now calls by name; drop them from the table: {named}"
    assert all(reason.strip() for reason in INDIRECT.values())
