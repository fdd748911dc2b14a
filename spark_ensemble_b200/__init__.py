"""spark_ensemble_b200 — H100-native (sm_90a) implementation of the row-parallel boosting hot path of
pierrenodet/spark-ensemble behind the reference's Estimator/Model surface.

    csrc/            hand-written CUDA kernels + the C ABI of include/se_abi.h (libse_b200.so)
    _native.py       ctypes binding of the C ABI (no fallback: raises when the library/GPU is missing)
    context.py       one GPU == one row shard (thin wrapper over se_ctx)
    gbm_engine.py    host driver of a GBM fit on a shard
    regression.py    GBMRegressor, GBMRegressionModel, BaggingRegressor(Model), BoostingRegressor(Model),
                     StackingRegressor(Model)
    classification.py GBMClassifier(Model), BoostingClassifier(Model), BaggingClassifier(Model),
                     StackingClassifier(Model)
    ensemble.py      DataFrame stand-in, HasSubBag.subspace, row partitioner, Dummy init models
    learners.py      base learners (third party in the reference; scikit-learn stand-ins here)
"""
__all__ = ["build", "Context", "DataFrame"]


def __getattr__(name):  # lazy: importing the package must not require the built library
    if name == "Context":
        from .context import Context
        return Context
    if name == "DataFrame":
        from .ensemble import DataFrame
        return DataFrame
    raise AttributeError(name)
