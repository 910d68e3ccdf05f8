"""CPU tier: the C-ABI library loads and exports every symbol include/garecon.h declares (no compute calls)."""
import ctypes
import re
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent


def test_library_exports_every_declared_symbol(garecon):
    import __graft_entry__ as ge
    path = ge.build_engine()
    lib = ctypes.CDLL(str(path))
    header = (REPO / "include" / "garecon.h").read_text()
    declared = set(re.findall(r"\b(gar_[a-z_0-9]+)\s*\(", header)) - {"gar_str"}
    assert declared == set(garecon.abi.EXPORTED_SYMBOLS)
    for sym in declared:
        assert getattr(lib, sym) is not None
    lib.gar_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.gar_version()


def test_engine_create_fails_loudly_without_a_gpu(garecon):
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    import pytest
    with pytest.raises(garecon.GarError) as ei:
        garecon.Engine()
    assert ei.value.rc == garecon.abi.GAR_E_NO_DEVICE


def test_ctypes_struct_sizes_match_header(garecon):
    # a drifted mirror would silently shift every pointer: pin sizes against a C compile of the header
    import subprocess, tempfile, textwrap
    src = textwrap.dedent('''
        #include <stdio.h>
        #include "garecon.h"
        int main(void) { printf("%zu %zu %zu %zu %zu\\n", sizeof(gar_objects), sizeof(gar_actual), sizeof(gar_changeset), sizeof(gar_op), sizeof(gar_config)); return 0; }
    ''')
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(REPO / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout.split()
    abi = garecon.abi
    assert [int(x) for x in out] == [ctypes.sizeof(abi.GarObjects), ctypes.sizeof(abi.GarActual), ctypes.sizeof(abi.GarChangeset), ctypes.sizeof(abi.GarOp), ctypes.sizeof(abi.GarConfig)]
