"""Generate tests/golden/gru_seq_golden.npz by running the UNMODIFIED reference ``RNNStateEncoder.seq_forward`` of
ss_baselines/av_nav/models/rnn_state_encoder.py (loaded as make_avnav_policy_golden.py loads it, from an upstream
sound-spaces checkout in ``SOUNDSPACES_REFERENCE``) in float64, forward and autograd backward.

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_gru_seq_golden.py

Per case ``<name>/<key>``: ``config`` (T, N, I, Hd); inputs ``x`` (T N, I), ``h0`` (1, N, Hd), ``masks`` (T N, 1),
the GRU's ``w_ih``, ``w_hh``, ``b_ih``, ``b_hh`` (set_params of tests/avnav_models.py) and the upstream gradients
``g_out`` / ``g_h_last``; outputs ``out`` and ``h_last``; the gradients ``dx``, ``dh0``, ``dw_ih``, ``dw_hh``,
``db_ih``, ``db_hh`` of sum(out g_out) + sum(h_last g_h_last).  The mask patterns are tests/gru_seq_models.CASES.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from avnav_models import set_params  # noqa: E402
from gru_seq_models import CASES, case_inputs  # noqa: E402
from make_avnav_policy_golden import load_reference  # noqa: E402


def main():
    rnn_cls = load_reference()[3]
    out = {}
    for i, (name, (T, N, I, Hd)) in enumerate(CASES.items()):
        ref = set_params(rnn_cls(I, Hd), seed=50 + i).double()
        x, h0, masks, g_out, g_h = case_inputs(name)
        x.requires_grad_(True)
        h0.requires_grad_(True)
        y, h_last = ref.seq_forward(x, h0, masks)
        ((y * g_out).sum() + (h_last * g_h).sum()).backward()
        rnn = ref.rnn
        out[f"{name}/config"] = np.array([T, N, I, Hd], np.int64)
        for k, v in (("x", x), ("h0", h0), ("masks", masks), ("g_out", g_out), ("g_h_last", g_h),
                     ("w_ih", rnn.weight_ih_l0), ("w_hh", rnn.weight_hh_l0), ("b_ih", rnn.bias_ih_l0),
                     ("b_hh", rnn.bias_hh_l0), ("out", y), ("h_last", h_last), ("dx", x.grad), ("dh0", h0.grad),
                     ("dw_ih", rnn.weight_ih_l0.grad), ("dw_hh", rnn.weight_hh_l0.grad),
                     ("db_ih", rnn.bias_ih_l0.grad), ("db_hh", rnn.bias_hh_l0.grad)):
            out[f"{name}/{k}"] = v.detach().numpy()
    dst = os.path.join(ROOT, "tests", "golden", "gru_seq_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
