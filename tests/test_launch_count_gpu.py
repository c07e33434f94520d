"""b200st_launch_count counts every kernel the library launches: each call below adds exactly the kernels it launches.
The refusal tests assert that a bad call launches nothing, which holds only if no launch goes uncounted."""
import pytest
import torch

from neurst_b200 import decode as D
from neurst_b200 import lib as L
from oracle import restatement as R
from tests import parity_utils as U

pytestmark = pytest.mark.gpu

SMALL = dict(model="speech", d=64, heads=4, enc_layers=2, dec_layers=2, ffn=128, channels=64, feat=80, in_channels=1, vocab=96)
BOS, EOS, UNK = 94, 95, 93


def _launches(call):
    before = L.launch_count()
    call()
    torch.cuda.synchronize()
    return L.launch_count() - before


@pytest.mark.parametrize("dtype,force_simt", [(torch.float32, False), (torch.bfloat16, False), (torch.float32, True)],
                         ids=["fp32", "bf16", "force_simt"])
def test_gemm_is_one_launch(dtype, force_simt):
    g = torch.Generator(device="cuda").manual_seed(0)
    A = torch.randn(128, 64, device="cuda", generator=g).to(dtype)
    B = torch.randn(96, 64, device="cuda", generator=g).to(dtype)
    C = torch.zeros(128, 96, device="cuda")
    assert _launches(lambda: L.gemm(A, B, C, force_simt=force_simt)) == 1
    ref = A.float() @ B.float().t()
    assert float((C - ref).abs().max() / ref.abs().max()) < 1e-2


def test_dropout_mask_is_one_launch():
    rt = U.speech_runtime(SMALL, "fp32")
    assert _launches(lambda: rt.dropout_mask("enc.0.self.attn", 1000, 0.1, 7)) == 1


def test_persistent_greedy_search_is_two_launches():
    P = U.chaotic_decode_params(R.init_params(SMALL, seed=0, random_bias=True), 4.0, 0)
    g = torch.Generator().manual_seed(0)
    src = torch.randn(2, 61, 80, 1, generator=g)
    lens = torch.tensor([61, 40])
    rt = U.speech_runtime(SMALL, "fp32")
    rt.load_parameters(P)
    enc, bias = D.encode(rt, dict(src=src, src_length=lens))
    cache = D.create_decoding_cache(rt, enc, bias, 24)
    torch.cuda.synchronize()
    # the initial state, then the whole search in one cooperative kernel
    n = _launches(lambda: D.greedy_search(rt, None, BOS, EOS, UNK, maximum_decode_length=24, extra_decode_length=8, cache=cache,
                                          persistent=True))
    assert int(rt.lib.b200st_greedy_used_graph()) == 2
    assert n == 2
