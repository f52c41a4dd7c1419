"""b200ddl - a Hopper (H100, sm_90a) native distributed deep-learning stack.

Capabilities mirror the notebook workflow of ``smellslikeml/distributed-deep-learning-workshop``
(see SURVEY.md): table ETL -> sharded loader -> Keras-like trainer -> Horovod-like distributed runtime ->
Hyperopt-like search -> MLflow-like tracking / registry / pyfunc -> batch inference, with the hot paths
(conv/BN/ReLU stack, optimizers, gradient all-reduce, input pipeline) written as sm_90a CUDA/C++.

Sub-packages are imported lazily so that ``import b200ddl`` stays cheap:

    b200ddl.Session                      session / namespace setup          (reference: 00_setup.py)
    b200ddl.data                         Catalog / Table ETL                (01_data_prep.py)
    b200ddl.loader                       converter + pinned ring loader     (Petastorm usage, 03_*.py)
    b200ddl.models                       build_model / preprocess / ResNet-50 engine / MobileNetV2
    b200ddl.train                        Trainer (compile/fit/evaluate/predict), callbacks, History
    b200ddl.optim                        fused SGD / Adam / Adadelta
    b200ddl.parallel (alias b200ddl.dist)  init/rank/size, Runner, DistributedOptimizer, callbacks
    b200ddl.hpo                          hp.*, fmin, tpe/rand, Trials, ParallelTrials
    b200ddl.tracking                     mlflow-like runs / params / metrics / artifacts / registry
    b200ddl.pyfunc                       PythonModel / log_model / load_model / shard_udf
    b200ddl.ops                          python entry points of the CUDA kernels
    b200ddl.utils                        timeline tracer, clocks sampler, misc
"""
import importlib as _importlib

__version__ = "0.1.0"

_SUBMODULES = ("data", "loader", "models", "train", "optim", "parallel", "hpo", "tracking", "pyfunc", "ops", "utils")
_ALIASES = {"dist": "parallel"}


def __getattr__(name):
    if name in _ALIASES:
        name = _ALIASES[name]
    if name in _SUBMODULES:
        return _importlib.import_module(__name__ + "." + name)
    if name == "Session":
        from .session import Session

        return Session
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
