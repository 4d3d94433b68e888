"""Writes tests/golden/rtf_client_symbols.txt: the FunASR C++ runtime symbols (mangled, sorted) that examples/offline_rtf_client.cpp
needs when it is compiled against the REFERENCE's own runtime/onnxruntime/include/funasrruntime.h -- the calls of
bin/funasr-onnx-offline-rtf.cpp: FunOfflineInit, the WFST decoder calls, CompileHotwordEmbedding, FunOfflineInfer and the result calls.
tests/test_offline_concurrent_host.py compiles the same client against this repository's include/funasrruntime_b200.h and requires
exactly these symbols, all exported by libfunasr_b200.so.
Run where the reference tree is present:  python oracle/make_rtf_client_symbols_golden.py <reference root>"""
import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(ROOT, "tests", "golden", "rtf_client_symbols.txt")
RUNTIME_SYMBOL = re.compile(r"^(_Z\d+)?(Fun|CompileHotwordEmbedding)")


def client_runtime_symbols(header, include_dir):
    """Undefined runtime symbols of the RTF client object compiled with FUNASR_RUNTIME_HEADER=header."""
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "client.o")
        subprocess.run(["g++", "-std=c++17", "-pthread", "-DFUNASR_RUNTIME_HEADER=" + header, "-I" + include_dir, "-I" + os.path.join(ROOT, "include"),
                        "-c", os.path.join(ROOT, "examples", "offline_rtf_client.cpp"), "-o", obj], check=True)
        out = subprocess.run(["nm", "-u", obj], check=True, stdout=subprocess.PIPE, text=True).stdout
    return sorted({ln.split()[-1] for ln in out.splitlines() if ln.strip() and RUNTIME_SYMBOL.match(ln.split()[-1])})


if __name__ == "__main__":
    ref = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("FUNASR_REFERENCE_ROOT")
    if not ref:
        sys.exit("usage: python oracle/make_rtf_client_symbols_golden.py <reference root>  (or set FUNASR_REFERENCE_ROOT)")
    syms = client_runtime_symbols('"funasrruntime.h"', os.path.join(ref, "runtime", "onnxruntime", "include"))
    with open(GOLDEN, "w") as f:
        f.write("\n".join(syms) + "\n")
    print("wrote", GOLDEN, len(syms), "symbols")
