"""Child process of tests/test_gpu_ransac_boundaries.py::test_batches_of_4096_and_4097: B2S_RANSAC_BATCH is read once per process,
so each batch size runs here.  Writes the result of the noisy pair of test_ransac_oracle_boundaries.py (5000 hypotheses, none of
which stops the loop) as JSON to argv[1]."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from open3d_slam_b200 import engine as E  # noqa: E402
from test_ransac_oracle_boundaries import NOISY_MAX, NOISY_PARAMS, noisy_pair  # noqa: E402


def params():
    return E.PlaceRecognitionParameters(ransacMaxCorrespondenceDistance=NOISY_PARAMS["max_corr"], ransacSeed=NOISY_PARAMS["seed"],
                                        ransacNumIter=NOISY_MAX)


def main(path):
    eng = E.Engine()
    sx, sf, tx, tf = noisy_pair()
    r = E.registrationRANSACBasedOnFeatureMatching(eng, eng.cloud(sx), eng.cloud(tx), E.Feature(eng, sf.T), E.Feature(eng, tf.T), params())
    out = dict(T=r.transformation_.ravel().tolist(), fitness=r.fitness_, rmse=r.inlier_rmse_, inliers=r.n_corr, hypotheses=r.hypotheses,
               validations=r.validations, best_hypothesis=r.best_hypothesis, n_feature_corr=r.n_feature_corr, used_mutual=r.used_mutual)
    with open(path, "w") as fh:
        json.dump(out, fh)
    eng.close()


if __name__ == "__main__":
    main(sys.argv[1])
