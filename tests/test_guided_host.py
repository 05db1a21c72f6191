"""Guided sampling on the CPU: the restatement the GPU tests compare against (tests/guided_oracle.py) checked on its own --
Philox4x32-10 against Random123's known-answer vectors, the draw rule's frequencies against q_j / (Q - sum_prev q), and
the log-probability's gradient against float64 autograd of the same formula and central finite differences."""
import numpy as np
import pytest
import torch

import guided_oracle as G

N = G.N


def test_philox_known_answers():
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        assert [int(x) for x in G.philox(ctr, key)] == list(want)


def _logits(seed, scale=1.0):
    return (np.random.default_rng(seed).standard_normal(N) * scale).astype(np.float32)


def test_table():
    l = _logits(1)
    w, q, cum, bad = G.table(l)
    assert not bad and abs(w.sum() - 1) < 1e-12
    assert np.array_equal(q, np.floor(w * 2.0 ** 31).astype(np.uint32))
    assert np.array_equal(cum, np.cumsum(q.astype(np.uint64)).astype(np.uint32)) and int(cum[-1]) < 2 ** 32
    l2 = l.copy(); l2[3:] = -np.inf
    assert G.table(l2)[3] and not G.table(np.where(np.arange(N) < 4, 0, -np.inf).astype(np.float32))[3]
    for v in (np.nan, np.inf):
        l3 = l.copy(); l3[7] = v
        assert G.table(l3)[3]


def test_draw_frequencies_chi_square():
    """Few cells with weight, so that the repeat rule matters: the joint frequency of the first two cells and of the
    third given them match q_j / (Q - sum_prev q) (chi-square over 10^5 seeded draws)."""
    from scipy.stats import chisquare
    l = np.full(N, -np.inf, np.float32)
    cells = [3, 77, 400, 401, 1599, 800]
    l[cells] = np.log(np.array([0.4, 0.2, 0.15, 0.1, 0.1, 0.05], np.float32))
    w, q, cum, bad = G.table(l)
    assert not bad
    K = 100000
    draws = np.array([G.draw(cum, 1305, 7, i) for i in range(K)])
    assert all(len(set(d)) == 4 for d in draws[:1000])
    qq = {c: float(q[c]) for c in cells}
    Q = sum(qq.values())
    pairs = [(a, b) for a in cells for b in cells if a != b]
    obs = np.array([np.sum((draws[:, 0] == a) & (draws[:, 1] == b)) for a, b in pairs])
    exp = np.array([qq[a] / Q * qq[b] / (Q - qq[a]) for a, b in pairs]) * K
    assert chisquare(obs, exp * obs.sum() / exp.sum()).pvalue > 1e-3
    sel = (draws[:, 0] == 3) & (draws[:, 1] == 77)
    rest = [c for c in cells if c not in (3, 77)]
    obs3 = np.array([np.sum(draws[sel, 2] == c) for c in rest])
    exp3 = np.array([qq[c] for c in rest]) / sum(qq[c] for c in rest) * sel.sum()
    assert chisquare(obs3, exp3).pvalue > 1e-3


def _torch_logp(logits, cands):
    w = torch.softmax(logits, 0)
    lp = logits.new_zeros(())
    for c in cands:
        S = logits.new_zeros(())
        for k in range(4):
            lp = lp + torch.log(w[c[k]]) - torch.log(1 - S)
            S = S + w[c[k]]
    return lp


@pytest.mark.parametrize("T", [1, 3])
def test_log_prob_gradient(T):
    l = _logits(2, 2.0)
    w, q, cum, _ = G.table(l)
    ncand = np.array([7, 0, 5][:T], np.int64)
    g = 11
    lp, grad = G.log_prob(w, cum, T, 1305, g, ncand)
    cands = [G.draw(cum, 1305, g * T + s, i) for s in range(T) for i in range(ncand[s])]
    lt = torch.tensor(l.astype(np.float64), requires_grad=True)
    ref = _torch_logp(lt, cands)
    ref.backward()
    assert abs(lp - ref.item()) <= 1e-12 * abs(ref.item())
    assert np.allclose(grad, lt.grad.numpy(), rtol=1e-12, atol=1e-12 * np.abs(grad).max())
    assert abs(grad.sum()) <= 1e-9 * np.abs(grad).max()
    # central finite differences of the same formula at the same cells (the draw is held fixed)
    h = 1e-6
    for j in list(np.unique(np.concatenate(cands))[:4]) + [100, 1000]:
        e = torch.zeros(N, dtype=torch.float64); e[j] = h
        base = torch.tensor(l.astype(np.float64))
        fd = (_torch_logp(base + e, cands) - _torch_logp(base - e, cands)).item() / (2 * h)
        assert abs(fd - grad[j]) <= 1e-6 * max(1.0, abs(grad[j]))
