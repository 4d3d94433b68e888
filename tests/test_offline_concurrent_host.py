"""CPU: examples/offline_rtf_client.cpp, N threads on one FunOfflineInit handle, links against the reference's runtime header."""
import os
import subprocess

import pytest

from conftest import ROOT


def test_rtf_client_links_against_the_reference_header(tmp_path):
    """examples/offline_rtf_client.cpp (the calls of bin/funasr-onnx-offline-rtf.cpp) compiled against include/funasrruntime_b200.h needs
    exactly the runtime symbols it needs against the reference's funasrruntime.h (tests/golden/rtf_client_symbols.txt,
    oracle/make_rtf_client_symbols_golden.py); the library exports them all, and the client links and fails cleanly without a model."""
    import shutil
    if shutil.which("g++") is None or shutil.which("nm") is None:
        pytest.skip("no g++ / nm")
    import make_rtf_client_symbols_golden as mk
    inc = os.path.join(ROOT, "include")
    with open(os.path.join(ROOT, "tests", "golden", "rtf_client_symbols.txt")) as f:
        want = f.read().split()
    assert len(want) == 11 and any("CompileHotwordEmbedding" in s for s in want)
    assert mk.client_runtime_symbols('"funasrruntime_b200.h"', inc) == want
    lib = os.path.join(ROOT, "funasr_b200", "libfunasr_b200.so")
    exported = {ln.split()[-1] for ln in subprocess.run(["nm", "-D", "--defined-only", lib], check=True, stdout=subprocess.PIPE,
                                                        text=True).stdout.splitlines() if ln.strip()}
    assert not [s for s in want if s not in exported]
    exe = str(tmp_path / "rtf_client")
    r = subprocess.run(["g++", "-std=c++17", "-pthread", '-DFUNASR_RUNTIME_HEADER="funasrruntime_b200.h"', "-I" + inc,
                        os.path.join(ROOT, "examples", "offline_rtf_client.cpp"), "-L" + os.path.join(ROOT, "funasr_b200"), "-lfunasr_b200",
                        "-Wl,-rpath," + os.path.join(ROOT, "funasr_b200"), "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    (tmp_path / "list.txt").write_text("a /nonexistent.wav\n")
    r = subprocess.run([exe, str(tmp_path), str(tmp_path / "list.txt"), "4"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 1 and "asr init failed" in r.stdout
