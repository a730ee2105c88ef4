"""Teacher-forced loss without a GPU: the labels forward(labels=...) hands to the kernels are the ones ForCausalLMLoss
([O] loss/loss_utils.py) compares the logits with, and a numpy restatement of the kernels' arithmetic (bf16-rounded logits,
128-column tile partials, a fixed-order merge) stays within the GPU tests' tolerance of the reference's loss."""
import numpy as np
import pytest
import torch

from audio_flamingo_b200.modeling import prepare_loss_labels


def _for_causal_lm_loss(logits, labels, V, **kw):
    from transformers.loss.loss_utils import ForCausalLMLoss

    return ForCausalLMLoss(logits, labels, V, **kw)


def _ours(logits, labels, V, shift_labels=None, ignore_index=-100, num_items_in_batch=None):
    """The loss from prepare_loss_labels, reduced as af3_lm_head_xent's totals are."""
    B, S = logits.shape[:2]
    lab = prepare_loss_labels(labels, shift_labels, ignore_index, B, S, V)
    nll = torch.nn.functional.cross_entropy(logits.reshape(-1, V).double(), lab, ignore_index=ignore_index, reduction="none")
    n = (lab != ignore_index).sum().double() if num_items_in_batch is None else torch.as_tensor(num_items_in_batch).double()
    return (nll.sum() / n).float()


def _case(seed, B=3, S=17, V=300):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, S, V, generator=g) * 3
    labels = torch.randint(0, V, (B, S), generator=g)
    labels[0, :4] = -100   # left padding
    labels[1, 7] = -100
    return logits, labels, V


@pytest.mark.parametrize("kw", [{}, {"ignore_index": 5}, {"num_items_in_batch": 29}, {"num_items_in_batch": torch.tensor(41)},
                                {"shift_labels": "roll"}, {"shift_labels": "roll", "num_items_in_batch": 7}])
def test_label_preparation_matches_for_causal_lm_loss(kw):
    logits, labels, V = _case(0)
    kw = dict(kw)
    if kw.get("shift_labels") == "roll":
        kw["shift_labels"] = torch.roll(labels, 2, dims=1)
    if "ignore_index" in kw:
        labels[labels == -100] = kw["ignore_index"]
        labels[2, 3:6] = kw["ignore_index"]
    ref = _for_causal_lm_loss(logits, labels, V, **kw)
    ours = _ours(logits, labels, V, **kw)
    assert torch.allclose(ours, ref, rtol=1e-6, atol=0), (ours, ref)


def test_shift_pads_right_and_moves_left_by_one():
    labels = torch.tensor([[-100, 4, 5, 6], [1, 2, 3, -100]])
    got = prepare_loss_labels(labels, None, -100, 2, 4, 10).view(2, 4)
    assert got.tolist() == [[4, 5, 6, -100], [2, 3, -100, -100]]
    got = prepare_loss_labels(labels.clamp(min=0), None, 9, 2, 4, 10).view(2, 4)
    assert got[:, -1].tolist() == [9, 9]
    sl = torch.tensor([[1, 2, 3, 4], [5, 6, 7, 8]], dtype=torch.int32)
    assert prepare_loss_labels(None, sl, -100, 2, 4, 10).tolist() == list(range(1, 9))


def test_all_ignored_is_nan_like_the_reference():
    logits, labels, V = _case(1)
    labels[:] = -100
    assert torch.isnan(_for_causal_lm_loss(logits, labels, V)) and torch.isnan(_ours(logits, labels, V))
    # with num_items_in_batch the reference's sum is 0
    assert _ours(logits, labels, V, num_items_in_batch=4) == _for_causal_lm_loss(logits, labels, V, num_items_in_batch=4) == 0


@pytest.mark.parametrize("bad", ["range_hi", "range_lo", "float", "bool", "shape", "ignore_index"])
def test_host_labels_are_validated(bad):
    labels = torch.randint(0, 10, (2, 5))
    kw = dict(shift_labels=None, ignore_index=-100, B=2, S=5, V=10)
    if bad == "range_hi":
        labels[1, 2] = 10
    elif bad == "range_lo":
        labels[0, 3] = -1
    elif bad == "float":
        labels = labels.float()
    elif bad == "bool":
        labels = labels > 3
    elif bad == "shape":
        labels = labels[:, :4]
    else:
        kw["ignore_index"] = -100.0
    with pytest.raises(ValueError):
        prepare_loss_labels(labels, **kw)
    # ignore_index itself may lie outside [0, V), and a label equal to it is fine wherever it is
    ok = torch.randint(0, 10, (2, 5))
    ok[0, 1] = -7
    prepare_loss_labels(ok, None, -7, 2, 5, 10)


def restate_kernel(logits32, labels, ignore_index=-100, tile=128):
    """af3_lm_head_xent in numpy: logits rounded to bf16; per 128-column tile (max, sum exp(v - max)) in fp32; the tiles
    merged in column order (max first, then the rescaled sums); nll = lse - logit[label] in fp32, 0 where uncounted."""
    T, V = logits32.shape
    v = torch.from_numpy(logits32).to(torch.bfloat16).float().numpy()
    n_ct = -(-V // tile)
    pad = np.full((T, n_ct * tile), -np.inf, dtype=np.float32)
    pad[:, :V] = v
    t = pad.reshape(T, n_ct, tile)
    m = t.max(-1)
    s = np.exp(t - m[..., None]).astype(np.float32).sum(-1, dtype=np.float32)
    M = m.max(-1)
    S = np.zeros(T, dtype=np.float32)
    for j in range(n_ct):
        S = (S + s[:, j] * np.exp(m[:, j] - M)).astype(np.float32)
    lse = (M + np.log(S)).astype(np.float32)
    counted = (labels != ignore_index) & (labels >= 0) & (labels < V)
    tgt = v[np.arange(T), np.where(counted, labels, 0)]
    return np.where(counted, lse - tgt, 0).astype(np.float32), counted


@pytest.mark.parametrize("V", [2048, 2051, 152064])
def test_kernel_restatement_matches_for_causal_lm_loss(V):
    rs = np.random.RandomState(V)
    T = 40 if V > 10000 else 300
    logits = (rs.randn(T, V) * 4).astype(np.float32)
    labels = rs.randint(0, V, size=T).astype(np.int64)
    labels[:3] = [0, V - 1, V - 2]   # first column, last column, tail tile when V % 128 != 0
    labels[5::7] = -100
    nll, counted = restate_kernel(logits, labels)
    # the reference on the same bf16-rounded logits, in fp64
    lb = torch.from_numpy(logits).to(torch.bfloat16).double()
    ref = torch.nn.functional.cross_entropy(lb, torch.from_numpy(labels), reduction="none").numpy()
    lse = torch.logsumexp(lb, -1).numpy()
    assert np.all(np.abs(nll - ref) <= 1e-5 * (1 + np.abs(lse))), np.abs(nll - ref).max()
    loss = nll.astype(np.float64).sum() / counted.sum()
    ref_loss = _for_causal_lm_loss(lb.float()[None], None, V, shift_labels=torch.from_numpy(labels)[None]).item()
    assert abs(loss - ref_loss) <= 1e-5 * (1 + np.abs(lse).max())
