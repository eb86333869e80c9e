"""The reference's answer loss and accuracy count, restated in its own form (boolean masks, per-batch counts) for the tests and
tools that check training.answer_loss and SplitEvalStep's scoring.  Pure torch; no GPU needed."""
import torch
import torch.nn.functional as F


def compute_loss(logits, labels, loss):
    """compute_loss of qagnn.py:208-224 on logits [bs, nc]: nn.CrossEntropyLoss, or nn.MarginRankingLoss(margin=0.1) on the
    correct logit of every question (repeated nc - 1 times) against its wrong logits, both selected from the flat logits
    with boolean masks built from the one-hot labels."""
    if loss == "cross_entropy":
        return torch.nn.CrossEntropyLoss(reduction="mean")(logits, labels)
    if loss != "margin_rank":
        raise ValueError(loss)
    nc = logits.size(1)
    flat = logits.view(-1)
    is_correct = F.one_hot(labels, num_classes=nc).view(-1)
    correct = flat[is_correct == 1].contiguous().view(-1, 1).expand(-1, nc - 1).contiguous().view(-1)
    wrong = flat[is_correct == 0]
    y = wrong.new_ones((wrong.size(0),))
    return torch.nn.MarginRankingLoss(margin=0.1, reduction="mean")(correct, wrong, y)


def evaluate_counts(logits, labels):
    """One batch of evaluate_accuracy (qagnn.py:30-38): (questions whose argmax is the label, questions), as ints."""
    return int((logits.argmax(1) == labels).sum().item()), int(labels.size(0))
