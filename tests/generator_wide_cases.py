"""Inputs and slices of the wide-map generator cases (tests/golden/make_generator_wide_golden.py and the tests that
read tests/golden/generator_wide.npz).  Helper module, not a test file."""
import os

from impersonator_b200 import synthetic

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "generator_wide.npz")
WIDTHS = (14, 18)               # 3 + the conditioning channels of 'par' (11) and 'binary' (15)


def sl(t, step=8):
    """Image / mask slice (NCHW)."""
    return t[:, :, 3::step, 5::step].contiguous().cpu().numpy()


def feat(t):
    """Feature-map slice (NCHW)."""
    return t[:, ::16, ::4, ::4].contiguous().cpu().numpy()


def stem_slice(t):
    """Slice of the stem's raw [B, 64, H, W] output."""
    return t[:, ::4, 3::8, 5::8].contiguous().cpu().numpy()


def cases(cin):
    """The inputs of every case of width cin."""
    return dict(front=synthetic.synthetic_generator_inputs(1, 256, seed=100 + cin, cin=cin),
                inf=synthetic.synthetic_generator_inputs(2, 256, seed=200 + cin, cin=cin),
                swap_a=synthetic.synthetic_generator_inputs(1, 256, seed=300 + cin, cin=cin),
                swap_b=synthetic.synthetic_generator_inputs(1, 256, seed=400 + cin, cin=cin),
                inf512=synthetic.synthetic_generator_inputs(1, 512, seed=500 + cin, cin=cin))


def weights(cin):
    """(ImpersonatorGenerator template from impersonator_b200.generator, fill_state_dict(seed=0)) for width cin."""
    from impersonator_b200.generator import ImpersonatorGenerator
    net = ImpersonatorGenerator(bg_dim=4, src_dim=cin, tsf_dim=cin, repeat_num=6)
    sd = synthetic.fill_state_dict(net.state_dict(), seed=0)
    net.load_state_dict(sd)
    return net, sd
