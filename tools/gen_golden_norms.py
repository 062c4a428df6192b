"""Whole-model golden vectors (Encodec.inference through the UNMODIFIED reference) for the `norm` / `causal` branches other than
{time_group_norm, non-causal}: conf/soundstream_16k_n32_600k_step.yaml's {weight_norm, causal, 3 dilated residual blocks, no
sequence model} and {weight_norm, non-causal, SLSTM}, at small widths.  Build container only:  python tools/gen_golden_norms.py"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from gen_golden import model_case  # noqa: E402

if __name__ == "__main__":
    model_case("soundstream_causal_small", 3, 3, 40 * 21 + 9, 41, bit_widths=(None,))
    model_case("weightnorm_lstm_small", 4, 2, 40 * 25 + 3, 42, bit_widths=(None, 8000))
    model_case("causal_lstm_small", 6, 2, 40 * 25, 43, bit_widths=(None,))      # {weight_norm, causal, SLSTM}
