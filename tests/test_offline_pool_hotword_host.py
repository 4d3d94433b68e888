"""CPU: the grouped hotword-memory entries (attention with a K/V entry per row, the contextual decoder and the SeACo stack over several
memories) are exported and declared, refuse bad maps, lengths and probe rows before any device work, and size their workspaces from
the same carve as the entries they extend."""
import ctypes as C

from funasr_b200 import _abi

NEW = ["fa_attention_grouped_workspace_bytes", "fa_attention_grouped", "fa_paraformer_decoder_grouped_workspace_bytes",
       "fa_paraformer_decoder_forward_grouped", "fa_sanm_decoder_stack_grouped_workspace_bytes", "fa_sanm_decoder_stack_forward_grouped"]
FAKE = C.c_void_p(256)                           # never dereferenced: every call below is refused first
BIG = 1 << 40


def _i32(v):
    return (C.c_int32 * len(v))(*v)


def test_new_symbols_exported_and_declared():
    lib = _abi.load()
    for name in NEW:
        assert name in _abi.SIGNATURES, name
        assert hasattr(lib, name), name


def _attn(lib, index, kv_batch=3, key_lens=FAKE, mode=3, head_dim=128):
    return lib.fa_attention_grouped(FAKE, 512, FAKE, 1024, FAKE, 1024, key_lens, index, kv_batch, 4, 4, head_dim, 5, 70, FAKE, 512, mode,
                                    FAKE, BIG, None)


def test_attention_grouped_refusals():
    lib = _abi.load()
    assert _attn(lib, None) == -1
    assert _attn(lib, _i32([0, 1, 2, 0]), key_lens=None) == -1
    assert _attn(lib, _i32([0, 1, 3, 0])) == -1                  # an index >= kv_batch
    assert _attn(lib, _i32([0, -1, 2, 0])) == -1
    assert _attn(lib, _i32([0, 0, 0, 0]), kv_batch=0) == -1
    assert _attn(lib, _i32([0, 1, 2, 0]), mode=7) == -1
    assert _attn(lib, _i32([0, 1, 2, 0]), head_dim=64) == -4     # the tensor cores take 128-wide heads


def _decoder(has_bias=1):
    d = _abi.FaDecoder()
    d.has_bias = has_bias
    return d


def _dec(lib, lens, groups, n_groups=2, nh_max=5, dec=None, embed=FAKE):
    dec = dec if dec is not None else _decoder()
    return lib.fa_paraformer_decoder_forward_grouped(C.byref(dec), FAKE, FAKE, 3, 40, FAKE, 9, FAKE, 9, FAKE, FAKE, None, 1, None, embed,
                                                     lens, groups, n_groups, nh_max, 3, FAKE, BIG, None)


def test_decoder_grouped_refusals():
    lib = _abi.load()
    ok_lens, ok_groups = [5, 2], [0, 1, 1]
    assert _dec(lib, None, _i32(ok_groups)) == -1
    assert _dec(lib, _i32(ok_lens), None) == -1
    assert _dec(lib, _i32(ok_lens), _i32([0, 2, 1])) == -1       # an index >= G
    assert _dec(lib, _i32(ok_lens), _i32([0, -1, 1])) == -1
    assert _dec(lib, _i32([0, 2]), _i32(ok_groups)) == -1        # a memory without rows
    assert _dec(lib, _i32([6, 2]), _i32(ok_groups)) == -1        # longer than nh_max
    assert _dec(lib, _i32(ok_lens), _i32(ok_groups), n_groups=0) == -1
    assert _dec(lib, _i32(ok_lens), _i32(ok_groups), embed=None) == -1
    assert _dec(lib, _i32(ok_lens), _i32(ok_groups), dec=_decoder(0)) == -1   # not a contextual decoder


def _stack(lib, lens, groups, probe, n_probe, probs=FAKE, n_groups=2, t_mem=5):
    d = _decoder(0)
    return lib.fa_sanm_decoder_stack_forward_grouped(C.byref(d), FAKE, lens, groups, n_groups, 3, t_mem, FAKE, 9, FAKE, 9, 6, 0, None, probs,
                                                     probe, n_probe, 3, FAKE, BIG, None)


def test_stack_grouped_refusals():
    lib = _abi.load()
    lens, groups = _i32([5, 2]), _i32([0, 1, 1])
    assert _stack(lib, None, groups, _i32([0]), 1) == -1
    assert _stack(lib, lens, None, _i32([0]), 1) == -1
    assert _stack(lib, lens, _i32([0, 2, 1]), _i32([0]), 1) == -1
    assert _stack(lib, _i32([0, 2]), groups, _i32([0]), 1) == -1
    assert _stack(lib, _i32([5, 6]), groups, _i32([0]), 1) == -1
    assert _stack(lib, lens, groups, _i32([0, 3]), 2) == -1       # a probed row >= batch
    assert _stack(lib, lens, groups, _i32([-1]), 1) == -1
    assert _stack(lib, lens, groups, None, 1) == -1
    assert _stack(lib, lens, groups, _i32([0]), 0) == -1


def test_workspace_queries_monotone_and_extend_the_existing_carves():
    lib = _abi.load()
    for m in (0, 1, 3):
        # one memory per row is the tensor-core carve of fa_attention_tc plus the index
        if m:
            assert lib.fa_attention_grouped_workspace_bytes(7, 4, 30, 7, 65, m) >= lib.fa_attention_tc_workspace_bytes(7, 4, 30, 65, m) + 28
        else:
            assert lib.fa_attention_grouped_workspace_bytes(7, 4, 30, 7, 65, m) == 256
        a = [lib.fa_attention_grouped_workspace_bytes(7, 4, 30, g, t, m) for g, t in ((1, 1), (1, 64), (3, 64), (3, 65), (7, 300))]
        assert a == sorted(a)
        # one memory: the existing contextual carve plus two ints per row
        for B, T, N, nh in ((3, 40, 9, 5), (8, 100, 30, 64)):
            one = lib.fa_paraformer_decoder_workspace_bytes_hw(B, T, N, 100, m, nh)
            assert lib.fa_paraformer_decoder_grouped_workspace_bytes(B, T, N, 100, m, 1, nh) >= one + 8 * B
            assert lib.fa_paraformer_decoder_grouped_workspace_bytes(B, T, N, 100, m, 1, nh) <= one + 8 * B + 256
        d = [lib.fa_paraformer_decoder_grouped_workspace_bytes(8, 100, 30, 100, m, g, nh) for g, nh in ((1, 1), (1, 50), (4, 50), (4, 65), (9, 300))]
        assert d == sorted(d)
        # the stack: one memory per row is the existing carve (which counts a per-row memory) plus the ints
        for B, t_mem, N in ((3, 5, 9), (8, 50, 30)):
            one = lib.fa_sanm_decoder_stack_workspace_bytes(B, t_mem, N, m)
            assert lib.fa_sanm_decoder_stack_grouped_workspace_bytes(B, B, t_mem, N, 0, m) >= one + 8 * B
        s = [lib.fa_sanm_decoder_stack_grouped_workspace_bytes(8, g, t, 30, p, m) for g, t, p in ((1, 1, 0), (1, 50, 1), (4, 50, 4), (9, 300, 8))]
        assert s == sorted(s)
    assert lib.fa_attention_grouped_workspace_bytes(0, 4, 30, 1, 64, 3) == 0
    assert lib.fa_sanm_decoder_stack_grouped_workspace_bytes(8, 0, 5, 30, 0, 3) == 0
