"""CPU: tests/optim_ref.py, the float64 update rules the GPU optimizer tests hold adam_kernel to, agrees with the
oracle's Adam and oracle/oracle_optim.py, and keeps the reference's edge rules (G's penalty quirk, sign(0) = 0, the
SGD first-evaluation clone, the accuracy history)."""
import numpy as np

import optim_ref as R
from oracle import oracle as O
from oracle import oracle_optim as OO


def _state(rng, n=1000):
    return (rng.standard_normal(n), rng.standard_normal(n) * 1e-2, rng.standard_normal(n) * 1e-3,
            rng.random(n) * 1e-5)


def test_adam_matches_oracle_over_resumed_steps():
    rng = np.random.default_rng(1)
    x, g, m, v = _state(rng)
    xo, mo, vo = x.copy(), m.copy(), v.copy()
    f = R.f32
    for t in (0, 1, 9999, 10 ** 6):
        x1, m1, v1, t1 = R.adam(x, g, m, v, t, 1e-3, 0.9, 0.999, 1e-8)
        O.f64.adam(xo, g, mo, vo, t + 1, f(1e-3), f(0.9), f(0.999), f(1e-8))
        assert t1 == t + 1
        np.testing.assert_allclose(m1, mo, rtol=1e-15, atol=1e-18)  # m may cancel: terms ~1e-3
        np.testing.assert_allclose(v1, vo, rtol=1e-15, atol=1e-21)
        np.testing.assert_allclose(x1, xo, rtol=1e-14, atol=1e-18)
        x, m, v = x1, m1, v1


def test_adagrad_and_sgd_match_oracle_optim():
    rng = np.random.default_rng(2)
    x, _, _, _ = _state(rng)
    for mom in (0.0, 0.5, 0.9):
        xs, xa, ref_s, ref_a = x.copy(), x.copy(), x.copy(), x.copy()
        buf, var = np.full_like(x, 123.0), np.zeros_like(x)  # the buffer a first SGD step must ignore
        st_s, st_a = {}, {}
        for t in range(4):
            g = rng.standard_normal(x.size)
            xs, buf, t_s = R.sgd(xs, g, buf, t, lr=0.02, mom=mom)
            xa, var, t_a = R.adagrad(xa, g, var, t, lr=1e-3)
            OO.sgd_step(ref_s, g, st_s, lr=R.f32(0.02), mom=R.f32(mom))
            OO.adagrad_step(ref_a, g, st_a, lr=R.f32(1e-3))
            assert t_s == t_a == st_s["evalCounter"] == t + 1
        np.testing.assert_allclose(xs, ref_s, rtol=1e-14, atol=1e-17)
        np.testing.assert_allclose(xa, ref_a, rtol=1e-14, atol=1e-17)
        if mom == 0:
            assert (buf == 123.0).all()


def test_penalty_quirk_sign_zero_and_clamp():
    p = np.array([0.0, -0.0, 2.0, -3.0, 0.5, 0.5])
    g = np.array([1.0, -1.0, 0.0, 0.0, 10.0, np.nan])
    l1, l2 = R.penalty_terms(False, 0.5, 0.25)  # G: the L1 term is weighted by G_L2
    assert (l1, l2) == (0.25, 0.25)
    assert R.penalty_terms(True, 0.5, 0.25) == (0.5, 0.25)
    assert R.penalty_terms(False, 0.0, 0.0) == (0.0, 0.0)
    out = R.consumed_grad(g, p, 0.5, l1, l2, clamp=1.0)
    # scale first, then sign(p)*l1 + p*l2 (sign(0) = 0), then the clamp; Torch's CPU clamp keeps a NaN
    np.testing.assert_array_equal(out[:5], [0.5, -0.5, 0.75, -1.0, 1.0])
    assert np.isnan(out[5])


def test_accuracy_gate_transcription():
    accs = []
    accs, go = R.accuracy_gate(accs, 0.5, 2, 0.6)
    assert go and accs == [0.5]
    accs, go = R.accuracy_gate(accs, 0.75, 2, 0.6)
    assert not go and accs == [0.5, 0.75]
    accs, go = R.accuracy_gate(accs, 0.25, 2, 0.6)  # the oldest falls out: mean(0.75, 0.25) = 0.5
    assert go and accs == [0.75, 0.25]
