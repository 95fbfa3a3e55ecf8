"""The k-NN evaluation protocol in float64 numpy (DINO / DINOv2 / DINOv3 k-NN): the statement the GPU kernels are
checked against.

Search: similarity = dot product; each query keeps its k nearest bank rows, similarity descending, ties to the lower
bank index.  Vote: for each k, weights softmax(sims[:k] / T); a class's score is the sum of the weights of its
neighbours among the first k; the 5 best classes, ties to the lower class index."""
import numpy as np


def topk(queries, bank, k):
    """(sims [Q, k] float64, idx [Q, k] int64, all_sims [Q, N])."""
    s = np.asarray(queries, np.float64) @ np.asarray(bank, np.float64).T
    idx = np.empty((s.shape[0], k), np.int64)
    for q in range(s.shape[0]):
        idx[q] = np.lexsort((np.arange(s.shape[1]), -s[q]))[:k]
    return np.take_along_axis(s, idx, 1), idx, s


def vote(sims, idx, labels, nb_knn, temperature, num_classes):
    """int64 [Q, len(nb_knn), 5] predictions (-1 past the number of classes)."""
    sims, labels = np.asarray(sims, np.float64), np.asarray(labels)
    out = np.empty((sims.shape[0], len(nb_knn), 5), np.int64)
    for q in range(sims.shape[0]):
        for t, k in enumerate(nb_knn):
            x = sims[q, :k] / temperature
            w = np.exp(x - x.max())
            w /= w.sum()
            scores = np.zeros(num_classes)
            for j in range(k):                       # neighbour order
                scores[labels[idx[q, j]]] += w[j]
            best = np.lexsort((np.arange(num_classes), -scores))[:5]
            out[q, t] = -1                           # fewer than 5 classes: the rest is -1
            out[q, t, :best.size] = best
    return out


def accuracy(preds, labels, nb_knn):
    """{k: {"top1", "top5"}} in percent."""
    y = np.asarray(labels).reshape(-1, 1)
    return {k: {"top1": 100.0 * float(np.mean(preds[:, t, 0] == y[:, 0])),
                "top5": 100.0 * float(np.mean((preds[:, t, :] == y).any(1)))} for t, k in enumerate(nb_knn)}
