"""Golden vectors for the xyz learning-rate schedule of PackedAdam, produced by CALLING THE REFERENCE'S OWN
get_expon_lr_func (gaussiansplatting/utils/general_utils.py:29-62).

    HUMANGAUSSIAN_ROOT=<HumanGaussian checkout> python tests/golden/make_golden_lr.py   ->  tests/golden/ref_lr.npz

Cases: the schedule GaussianModel.training_setup builds from the reference's OptimizationParams defaults
(gaussiansplatting/arguments/__init__.py:73-76, spatial_lr_scale 1; gaussian_model.py:166-169), and a delayed variant
(lr_delay_steps > 0) that exercises the reverse-cosine warm-up.  Each is evaluated at a few hundred steps, including
step < 0, step 0, the delay window and steps past max_steps.  The tests only read the fixture.
"""
import os
import sys

import numpy as np

REF = os.environ["HUMANGAUSSIAN_ROOT"]
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)

CASES = {
    # lr_init, lr_final, lr_delay_steps, lr_delay_mult, max_steps
    "default": (0.00005, 0.000025, 0, 0.5, 30_000),
    "delayed": (0.00016, 0.0000016, 500, 0.01, 30_000),
}


def main():
    from gaussiansplatting.utils import general_utils
    steps = np.unique(np.concatenate([[-5, -1], np.arange(0, 40), np.arange(40, 1200, 13), np.linspace(1200, 40_000, 150).astype(np.int64)]))
    out = {"steps": steps.astype(np.int64)}
    for name, (lr_init, lr_final, delay_steps, delay_mult, max_steps) in CASES.items():
        f = general_utils.get_expon_lr_func(lr_init=lr_init, lr_final=lr_final, lr_delay_steps=delay_steps, lr_delay_mult=delay_mult,
                                            max_steps=max_steps)
        out[f"{name}_args"] = np.array([lr_init, lr_final, delay_steps, delay_mult, max_steps], np.float64)
        out[f"{name}_lr"] = np.array([float(f(int(s))) for s in steps], np.float64)
    np.savez_compressed(os.path.join(HERE, "ref_lr.npz"), **out)
    print("wrote ref_lr.npz:", len(steps), "steps per case")


if __name__ == "__main__":
    main()
