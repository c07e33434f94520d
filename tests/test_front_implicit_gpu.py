"""Speech front-end parity at the shapes where the implicit conv2 GEMMs change how they tile the parity-class planes, which
the feature sizes of test_speech_front_gpu.py do not reach.

In 16 bits with C == 256, Cin == 1 and F2 <= 128, conv2's forward and filter gradient read conv1's post-activation from
four parity-class planes.  The filter gradient's k-block is a chunk of whole time rows of one utterance: 64 // F2 rows
while F2 <= 64, the rest of the 64 k rows held at zero in both operands; one row in two halves of 64 frequencies when
64 < F2 <= 128, the second half partly past the tensor.  The forward's row tile is 128 // F2 time rows, remapped to the
dense rows of z2.

  F=256: F2 = 64, one full row per k-block (no zero rows), tu = 2
  F=257: F2 = 65 (F1 = 129 odd), two halves per row, the second one frequency wide, tu = 1
  F=131: F2 = 33, one row per k-block and 31 zero rows (the most), tu = 3
  F=127: F2 = 32 (F1 = 64 even), two rows per k-block, tu = 4
  F=5:   F2 = 2 (F1 = 3 odd), 32 rows per k-block, tu = 64

Each at one odd and one even T1; at F=127 and F=5 one of the two leaves the last k-block of an utterance partly past T2."""
import pytest

from tests.test_speech_front_gpu import check, front_errors

pytestmark = pytest.mark.gpu

#        F: (T with odd T1, T with even T1)
FEATS = {256: (9, 12), 257: (9, 12), 131: (45, 52), 127: (45, 52), 5: (261, 260)}
CASES = [(F, T, probe) for F, ts in FEATS.items() for T in ts for probe in ("random", "t_end", "f_end", "start")]


@pytest.mark.parametrize("F,T,probe", CASES)
def test_front_implicit_fp16_vs_oracle(F, T, probe):
    check(front_errors(F, 256, 1, T, "fp16", probe), "fp16")


@pytest.mark.parametrize("F,T", [(F, T) for F, ts in FEATS.items() for T in ts])
def test_front_implicit_bf16_vs_oracle(F, T):
    check(front_errors(F, 256, 1, T, "bf16", "random"), "bf16")
