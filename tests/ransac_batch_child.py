"""Child process of tests/test_gpu_place_recognition.py::test_batch_size_does_not_change_the_result: B2S_RANSAC_BATCH is read once
per process, so each batch size runs here.  Writes the results of a constructed two-target call as JSON to argv[1]; inputs() is shared with the test."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402

from open3d_slam_b200 import engine as E  # noqa: E402
from test_ransac_oracle import pair, rigid  # noqa: E402


def inputs():
    """one source against two targets (the second with its features reversed, so its correspondence set differs); half the
    source points do not match their targets' geometry, so the confidence rule spans several batches of a small B"""
    T = rigid(-0.5, [2.0, 1.0, 0.0])
    sx, sf, tx, tf = pair(300, T, 4)
    sx[150:] = np.random.default_rng(8).uniform(-10, 10, (150, 3))
    pr = E.PlaceRecognitionParameters(ransacMaxCorrespondenceDistance=0.3, ransacSeed=3, ransacNumIter=2000)   # target 2 runs to the cap
    return sx, sf, [(tx, tf), (tx + [0.0, 0.0, 5.0], tf[::-1].copy())], pr


def main(path):
    eng = E.Engine()
    sx, sf, targets, pr = inputs()
    f = lambda a: E.Feature(eng, a.T)
    rs = E.registrationRANSACBasedOnFeatureMatchingBatch(eng, eng.cloud(sx), [eng.cloud(x) for x, _ in targets], f(sf),
                                                         [f(t) for _, t in targets], pr)
    out = [dict(T=r.transformation_.ravel().tolist(), fitness=r.fitness_, rmse=r.inlier_rmse_, inliers=r.n_corr, hypotheses=r.hypotheses,
                validations=r.validations, best_hypothesis=r.best_hypothesis, n_feature_corr=r.n_feature_corr, used_mutual=r.used_mutual)
           for r in rs]
    with open(path, "w") as fh:
        json.dump(out, fh)
    eng.close()


if __name__ == "__main__":
    main(sys.argv[1])
