"""CPU checks of the C-ABI library: it builds for sm_90a, loads, and exports every declared symbol."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    sys.path.insert(0, ROOT)
    import __graft_entry__
    return __graft_entry__.build()


def test_library_loads_and_exports_all_declared_symbols(built_lib):
    from medaka_b200 import libmedaka as lm
    lib = lm.load()
    names = lm.declared_functions()
    assert len(names) >= 30
    for name in names:
        assert getattr(lib, name) is not None, name
    out = subprocess.run(["nm", "-D", "--defined-only", built_lib], capture_output=True, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in names:
        assert name in exported, name


def test_constants_match_reference_library():
    # libmedaka.lib.plp_bases / featlen / fwd_del / rev_del  (src/medaka_counts.h:19-22)
    from medaka_b200 import libmedaka as lm
    lib = lm.load()
    assert lm.ffi.string(lib.mdk_plp_bases()) == b"acgtACGTdD"
    assert (lib.mdk_featlen(), lib.mdk_fwd_del(), lib.mdk_rev_del()) == (10, 9, 8)
    assert lib.MDK_PREC_TC == 0 and lib.MDK_NORM_FWD_REV == 1


def test_preferred_windows_is_one_wave():
    # 16 windows per tile x (132 SMs of an H100 / 2 directions): host logic only, no device needed
    from medaka_b200 import libmedaka as lm
    lib = lm.load()
    assert lib.mdk_engine_preferred_windows(lm.ffi.NULL) == 16 * 66


def test_layout_helpers_host(tmp_path):
    """tiled_row / gi_quad_index (the layouts every tensor-core kernel agrees on) are bijections with the block structure
    the kernels rely on: host-only C++ property check compiled with nvcc."""
    import __graft_entry__
    exe = str(tmp_path / "layout_check")
    src = os.path.join(ROOT, "tests", "native", "layout_check.cu")
    subprocess.run([__graft_entry__._nvcc(), "-std=c++17", "-O1", "-o", exe, src], check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def test_sass_contains_wgmma_and_bulk_copy(built_lib):
    """The tensor-core kernels really are wgmma (HGMMA) with TMA-engine bulk copies (UBLKCP)."""
    sass = subprocess.run(["cuobjdump", "-sass", built_lib], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA", "UBLKCP", "SYNCS"):
        assert mnemonic in sass, mnemonic
    assert "UTCHMMA" not in sass


def test_no_cpu_fallback_without_gpu():
    from medaka_b200 import libmedaka as lm
    from medaka_b200 import models
    if lm.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(lm.MedakaB200Error):
        models.GRUModel()


def test_product_package_does_not_import_oracle():
    pkg = os.path.join(ROOT, "medaka_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f
