"""Loader of oracle/_ref/libstampsent_ref.so: the C++ runtime's own TimestampSentence (runtime/onnxruntime/src/util.cpp:569-637),
compiled by oracle/stampsent/Makefile from the reference tree where it is present.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "_ref", "libstampsent_ref.so")
REFERENCE_ROOT = os.environ.get("FUNASR_REFERENCE_ROOT", "/root/reference")


def build(force: bool = False) -> bool:
    """Compile from the reference tree when it is present; elsewhere use a prebuilt file if there is one."""
    if os.path.exists(SO) and not force:
        return True
    if not os.path.isfile(os.path.join(REFERENCE_ROOT, "runtime", "onnxruntime", "src", "util.cpp")):
        return False
    r = subprocess.run(["make", "-C", os.path.join(HERE, "stampsent"), "REF=" + REFERENCE_ROOT] + (["-B"] if force else []),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/stampsent build failed:\n" + r.stdout[-2000:])
    return os.path.exists(SO)


_lib = None


def timestamp_sentence(text: str, stamp: str) -> str:
    global _lib
    if _lib is None:
        _lib = C.CDLL(SO)
        _lib.stampsent_ref.restype = C.c_int
        _lib.stampsent_ref.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
    cap = 4096
    while True:
        buf = C.create_string_buffer(cap)
        n = _lib.stampsent_ref(text.encode("utf-8"), stamp.encode("utf-8"), buf, cap)
        if n >= 0:
            return buf.raw[:n].decode("utf-8", errors="surrogateescape")
        cap = -n + 1
