"""Host side of the one-token decode step: the split planner of `attn_decode`, its workspace size, the ABI, and the refusals of
`generate(use_cuda_graph=True)`.  No GPU needed."""
import ctypes

import pytest
import torch


def _plan(B, nkv, max_len, sms):
    from dreamllm_b200 import _lib
    ns, sl = ctypes.c_int(0), ctypes.c_int(0)
    assert _lib.lib().dllm_attn_decode_plan(B, nkv, max_len, sms, ctypes.byref(ns), ctypes.byref(sl)) == 0
    return ns.value, sl.value


@pytest.mark.parametrize("B", [1, 5, 8, 32])
@pytest.mark.parametrize("nkv", [32, 8, 4, 1])
@pytest.mark.parametrize("sms", [132, 114, 1])
def test_decode_split_plan(B, nkv, sms):
    from dreamllm_b200 import _lib
    lens = set()
    for max_len in (1, 63, 64, 65, 513, 2048, 2112, 4096, 32768):
        ns, sl = _plan(B, nkv, max_len, sms)
        lens.add(sl)
        assert sl % 64 == 0 and sl >= 64
        assert ns * sl >= max_len, "the splits cover the cache"
        assert (ns - 1) * sl < max_len, "no split is empty at kv_len = max_len"
        for nh in (nkv, 4 * nkv):
            for d in (64, 128):
                want = ns * B * nh * (d + 2) * 4
                assert _lib.lib().dllm_attn_decode_workspace_bytes(B, nh, nkv, d, max_len, sms) == want
        assert _plan(B, nkv, max_len, sms) == (ns, sl)
    assert len(lens) == 1, "the split length depends on (B, nkv, SMs) only, so the bits do not depend on max_len"


def test_decode_abi_signatures():
    from dreamllm_b200 import _lib
    L = _lib.lib()
    for name in ("dllm_attn_decode_plan", "dllm_attn_decode_workspace_bytes", "dllm_attn_decode", "dllm_rope_append_kv"):
        assert name in _lib.SIGNATURES
        fn = getattr(L, name)
        assert fn.argtypes == _lib.SIGNATURES[name][1] and fn.restype == _lib.SIGNATURES[name][0]
    assert len(_lib.SIGNATURES["dllm_attn_decode"][1]) == 19 and len(_lib.SIGNATURES["dllm_rope_append_kv"][1]) == 14
    # bad shapes are refused before anything touches a device
    assert L.dllm_attn_decode_plan(0, 8, 64, 132, ctypes.byref(ctypes.c_int()), ctypes.byref(ctypes.c_int())) != 0
    assert L.dllm_attn_decode(None, 0, None, None, None, None, 0, None, 0, None, 0, 1, 64, 12, 4, 128, 0.1, 132, None) == -6  # group 3
    assert L.dllm_attn_decode(None, 0, None, None, None, None, 0, None, 0, None, 0, 1, 64, 8, 8, 96, 0.1, 132, None) == -6   # d 96


class _Cfg:
    def __init__(self, **kw):
        self.__dict__.update(kw)


class _Model:
    def __init__(self, **cfg):
        self.config = _Cfg(**cfg)
        self.called = False

    def __call__(self, **kw):
        self.called = True
        raise AssertionError("the prefill must not run")


@pytest.mark.parametrize("flag", ["output_attentions", "log_attentions"])
def test_graph_decode_refuses_attention_outputs(flag):
    from dreamllm_b200.generation import beam_search, generate
    ids = torch.zeros(1, 4, dtype=torch.long)
    for fn in (generate, beam_search):
        m = _Model(**{flag: True})
        with pytest.raises(ValueError, match="output_attentions"):
            fn(m, ids, max_new_tokens=2, use_cuda_graph=True)
        assert not m.called
