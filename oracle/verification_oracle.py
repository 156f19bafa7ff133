"""CPU restatement of the reference's verification metric — TEST INFRASTRUCTURE ONLY.

* 8-crop distance averaging of the test loop, reference train_triplet.py:339-350;
* best-threshold accuracy sweep, reference eval_metrics.py:5-50 (thresholds 0..30 step 0.01);
* equal error rate: the reference has NO EER function (SURVEY §2, §8f); it is derived here from the same
  threshold sweep as the point where false-accept rate == false-reject rate (linear interpolation).
"""
import numpy as np


def crop_mean_distances(dists, n_pairs, crops):
    """train_triplet.py:350: dists.reshape(current_sample, test_input_per_file).mean(axis=1)"""
    return np.asarray(dists).reshape(n_pairs, crops).mean(axis=1)


def calculate_accuracy(threshold, dist, actual_issame):
    """eval_metrics.py:40-50"""
    predict_issame = np.less(dist, threshold)
    tp = np.sum(np.logical_and(predict_issame, actual_issame))
    fp = np.sum(np.logical_and(predict_issame, np.logical_not(actual_issame)))
    tn = np.sum(np.logical_and(np.logical_not(predict_issame), np.logical_not(actual_issame)))
    fn = np.sum(np.logical_and(np.logical_not(predict_issame), actual_issame))
    tpr = 0 if (tp + fn == 0) else float(tp) / float(tp + fn)
    fpr = 0 if (fp + tn == 0) else float(fp) / float(fp + tn)
    acc = float(tp + tn) / dist.size
    return tpr, fpr, acc


def calculate_roc(thresholds, distances, labels):
    """eval_metrics.py:16-37: (tpr, fpr, accuracy) at the threshold with the best accuracy (first argmax)."""
    res = np.array([calculate_accuracy(t, distances, labels) for t in thresholds])
    best = int(np.argmax(res[:, 2]))
    return res[best, 0], res[best, 1], res[best, 2]


def evaluate_accuracy(distances, labels):
    """eval_metrics.py:5-9 (the VAL@FAR half of evaluate() is not on the path under test)."""
    return calculate_roc(np.arange(0, 30, 0.01), np.asarray(distances), np.asarray(labels).astype(bool))


def equal_error_rate(distances, labels, thresholds=None):
    """Derived metric: FAR(t) = P(d < t | different), FRR(t) = P(d >= t | same); EER where they cross."""
    d = np.asarray(distances, dtype=np.float64)
    same = np.asarray(labels).astype(bool)
    if thresholds is None:
        thresholds = np.arange(0, 30, 0.01)
    far = np.array([(d[~same] < t).mean() for t in thresholds])
    frr = np.array([(d[same] >= t).mean() for t in thresholds])
    diff = far - frr
    i = int(np.argmax(diff >= 0))
    if i == 0:
        return float((far[0] + frr[0]) / 2)
    # linear interpolation between the bracketing thresholds
    w = -diff[i - 1] / (diff[i] - diff[i - 1]) if diff[i] != diff[i - 1] else 0.0
    return float((far[i - 1] + w * (far[i] - far[i - 1]) + frr[i - 1] + w * (frr[i] - frr[i - 1])) / 2)


def calculate_val_far(threshold, dist, actual_issame):
    """eval_metrics.py:75-88"""
    predict_issame = np.less(dist, threshold)
    true_accept = np.sum(np.logical_and(predict_issame, actual_issame))
    false_accept = np.sum(np.logical_and(predict_issame, np.logical_not(actual_issame)))
    n_same = np.sum(actual_issame)
    n_diff = np.sum(np.logical_not(actual_issame))
    if n_diff == 0:
        n_diff = 1
    if n_same == 0:
        return 0, 0
    return float(true_accept) / float(n_same), float(false_accept) / float(n_diff)


def calculate_val(thresholds, distances, labels, far_target=0.1):
    """eval_metrics.py:53-73.  The reference's scipy interp1d('slinear') call raises on the duplicate FAR values of any
    real curve under current scipy (tools/make_golden.py records the failure), so the crossing threshold is pinned on
    the de-duplicated curve, where 'slinear' is plain linear interpolation: the golden `val_threshold_dedup` is produced
    by the reference's OWN interp1d call on that curve."""
    far_train = np.array([calculate_val_far(t, distances, labels)[1] for t in thresholds])
    if np.max(far_train) >= far_target:
        keep = np.concatenate(([True], np.diff(far_train) > 0))
        x, y = far_train[keep], thresholds[keep]
        threshold = float(y[0]) if far_target <= x[0] else float(np.interp(far_target, x, y))
    else:
        threshold = 0.0
    val, far = calculate_val_far(threshold, distances, labels)
    return val, far, threshold
