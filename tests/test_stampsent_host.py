"""CPU: tests/stampsent_ref.py (the Python restatement of the C++ runtime's TimestampSentence, what FunASRGetStampSents returns)
against the committed golden of the compiled reference and, where it is built, against oracle/_ref/libstampsent_ref.so itself on
random (text, stamp) pairs: mismatched counts, texts without punctuation, 2- and 4-byte characters, empty stamps."""
import os

import numpy as np

from conftest import GOLDEN

import stampsent_lib
import stampsent_ref as S
from stampsent_cases import pairs


def test_restatement_equals_the_golden_of_the_compiled_reference():
    g = np.load(os.path.join(GOLDEN, "stampsent_cases.npz"))
    assert len(g["sents"]) >= 500 and sum(str(o) != "[]" for o in g["sents"]) > 200
    for t, s, o in zip(g["text"], g["stamp"], g["sents"]):
        assert S.timestamp_sentence(str(t), str(s)) == str(o), (str(t), str(s))


def test_restatement_equals_the_compiled_reference():
    if not stampsent_lib.build():
        import pytest
        pytest.skip("oracle/_ref/libstampsent_ref.so not built (no reference tree); the golden covers it")
    for t, s in pairs(99, 2000) + [("", ""), ("你好", ""), ("你好", "[[0,10],[10,20]]"), ("你好。", "[[0,10]]"), ("。", "[[0,1]]")]:
        assert S.timestamp_sentence(t, s) == stampsent_lib.timestamp_sentence(t, s), (t, s)


def test_hand_made_cases():
    # the full-width comma U+FF0C lies outside the runtime's punctuation ranges: it is glued to the next Latin word, as the runtime does
    assert S.timestamp_sentence("你好，world。", "[[0,100],[100,200],[200,400]]") == (
        '[{"text_seg":"你 好 ，world","punc":"。","start":0,"end":400,"ts_list":[[0,100],[100,200],[200,400]]}]')
    assert S.timestamp_sentence("你好、world。", "[[0,100],[100,200],[200,400]]") == (
        '[{"text_seg":"你 好","punc":"、","start":0,"end":200,"ts_list":[[0,100],[100,200]]},'
        '{"text_seg":"world","punc":"。","start":200,"end":400,"ts_list":[[200,400]]}]')
    assert S.timestamp_sentence("你好", "[[0,100],[100,200]]") == '[{"text_seg":"你 好","punc":"","start":0,"end":200,"ts_list":[[0,100],[100,200]]}]'
    assert S.timestamp_sentence("", "") == "[]"
