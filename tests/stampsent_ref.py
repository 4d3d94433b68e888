"""Python restatement of the C++ runtime's TimestampSentence (runtime/onnxruntime/src/util.cpp:569-637) -- the sentence list that
FunASRGetStampSents returns -- with the helpers it calls: TimestampSplitChiEngCharacters (:320-364) over EncodeConverter's UTF-8 ->
UTF-16 decoding (encode_converter.cpp:201-327: 3-byte and 2-byte sequences only; any other byte, a 4-byte sequence included, becomes
one 0 unit, which contributes nothing), both TimestampIsPunctuation overloads (:257-266 bytewise, :307-318 per unit), ParseTimestamps
and VectorToString.  Pinned against the compiled reference (oracle/_ref/libstampsent_ref.so) and tests/golden/stampsent_cases.npz;
the runtime shim's C++ (csrc/runtime_shim.cpp) is checked against this on the GPU."""
from typing import List

_PUNC_BYTES = set("，。？、,?".encode("utf-8"))


def _units(text: str) -> List[int]:
    b = text.encode("utf-8", errors="surrogateescape")
    out, i, n = [], 0, len(b)
    while i < n:
        c = b[i]
        if (c & 0xF0) == 0xE0 and n - i >= 3:
            if (b[i + 1] & 0xC0) == 0x80 and (b[i + 2] & 0xC0) == 0x80:
                u = ((c & 0x0F) << 12) | ((b[i + 1] & 0x3F) << 6) | (b[i + 2] & 0x3F)
                out.append(u if u >= 0x800 else 0)
                i += 3 if u >= 0x800 else 1
            else:
                out.append(0)
                i += 1
        elif (c & 0xE0) == 0xC0 and n - i >= 2:
            if (b[i + 1] & 0xC0) == 0x80:
                u = ((c & 0x1F) << 6) | (b[i + 1] & 0x3F)
                out.append(u if 0x80 <= u <= 0x7FF else 0)
                i += 2 if 0x80 <= u <= 0x7FF else 1
            else:
                out.append(0)
                i += 1
        else:
            out.append(c if c < 0x80 else 0)
            i += 1
    return out


def _unit_punc(u: int) -> bool:
    if u in (0x26, 0x27, 0x2D):
        return False
    return 0x21 <= u <= 0x2F or 0x3A <= u <= 0x40 or 0x5B <= u <= 0x60 or 0x7B <= u <= 0x7E or 0x2000 <= u <= 0x206F or 0x3000 <= u <= 0x303F


def split_chi_eng(text: str) -> List[str]:
    chars, eng = [], ""
    for u in _units(text):
        if 0x4E00 <= u <= 0x9FFF or 0x3400 <= u <= 0x4DFF or 0x30 <= u <= 0x39 or _unit_punc(u):
            if eng:
                chars.append(eng)
                eng = ""
            chars.append(chr(u))
        elif u == 0x20:
            if eng:
                chars.append(eng)
                eng = ""
        elif u != 0:
            eng += chr(u)
    if eng:
        chars.append(eng)
    return chars


def is_punctuation(s: str) -> bool:
    return all(c in _PUNC_BYTES for c in s.encode("utf-8"))


def parse_timestamps(s: str) -> List[List[int]]:
    """ParseTimestamps for the well-formed "[[b,e],[b,e],...]" strings FunASRGetStamp returns ("" and "[]" give none)."""
    if len(s) <= 2:
        return []
    out = []
    for seg in s[1:].split("]"):
        if seg in ("", ","):
            continue
        parts = seg.lstrip(",").lstrip("[").split(",")
        if len(parts) != 2:
            return []
        out.append([int(parts[0]), int(parts[1])])
    return out


def vector_to_string(v: List[List[int]]) -> str:
    return "[" + ",".join("[" + ",".join(str(x) for x in p) + "]" for p in v) + "]"


def timestamp_sentence(text: str, stamp: str) -> str:
    chars = split_chi_eng(text)
    ts = parse_timestamps(stamp)
    idx_ts, start, end = 0, -1, -1
    text_seg, out, seg = "", "", []
    for i, c in enumerate(chars):
        if is_punctuation(c):
            if seg:
                start, end = seg[0][0], seg[-1][1]
            sent = '{"text_seg":"%s","punc":"%s","start":%d,"end":%d,"ts_list":%s}' % (text_seg, c, start, end, vector_to_string(seg))
            out += sent if i == len(chars) - 1 else sent + ","
            text_seg, start, end, seg = "", 0, 0, []
        elif idx_ts < len(ts):
            text_seg = c if not text_seg else text_seg + " " + c
            seg.append(ts[idx_ts])
            idx_ts += 1
    if seg:
        start, end = seg[0][0], seg[-1][1]
        out += '{"text_seg":"%s","punc":"","start":%d,"end":%d,"ts_list":%s}' % (text_seg, start, end, vector_to_string(seg))
    return "[" + out + "]"
