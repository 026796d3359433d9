"""spark-agd_b200: H100-native accelerated (proximal) gradient descent -- the hot path of
staple/spark-agd (AcceleratedGradientDescent.optimize) behind the reference's own operator API.

Layout: csrc/ holds the sm_90a CUDA kernels and the C-ABI (include/agd_b200.h); optimization.py is
the host-side mirror of the reference interface.  The directory name carries a hyphen (the repo's
naming contract); import it as `spark_agd_b200` through the loader module at the repo root.
"""
from . import _native
from ._native import NativeError, build, exported_symbols
from .glm import (GeneralizedLinearAlgorithm, GeneralizedLinearModel, LinearRegressionModel, LinearRegressionWithAGD,
                  LogisticRegressionModel, LogisticRegressionWithAGD, SVMModel, SVMWithAGD, append_bias, column_std)
from .optimization import (DEFAULT_SPLIT_SEED, AcceleratedGradientDescent, Context, DeviceDataset, Evaluation, Gradient, GradientDescent,
                           HingeGradient, L1Updater, LeastSquaresGradient, LogisticGradient, MLUtils, RunStats,
                           SimpleUpdater, SquaredL2Updater, Updater, bf16_to_f32, physical_model, physical_projection, run_with_stats,
                           split_bounds)
from .stat import MultivariateStatisticalSummary, Statistics
from .feature import StandardScaler, StandardScalerModel
from .evaluation import BinaryClassificationMetrics, MulticlassMetrics
from .linalg import RowMatrix, SingularValueDecomposition
from .clustering import KMeans, KMeansModel, LocalKMeans
from .classification import NaiveBayes, NaiveBayesModel

__all__ = ["GeneralizedLinearAlgorithm", "GeneralizedLinearModel", "LinearRegressionModel", "LinearRegressionWithAGD",
           "LogisticRegressionModel", "LogisticRegressionWithAGD", "SVMModel", "SVMWithAGD",
           "append_bias", "column_std", "AcceleratedGradientDescent", "Context", "DeviceDataset", "Evaluation", "Gradient",
           "GradientDescent",
           "HingeGradient", "L1Updater", "LeastSquaresGradient", "LogisticGradient", "MLUtils", "NativeError", "RunStats",
           "SimpleUpdater", "SquaredL2Updater", "Updater", "bf16_to_f32", "build", "exported_symbols", "run_with_stats",
           "DEFAULT_SPLIT_SEED", "split_bounds", "MultivariateStatisticalSummary", "Statistics", "StandardScaler",
           "StandardScalerModel", "physical_model", "physical_projection", "BinaryClassificationMetrics", "RowMatrix",
           "SingularValueDecomposition", "KMeans", "KMeansModel", "LocalKMeans", "NaiveBayes", "NaiveBayesModel",
           "MulticlassMetrics"]
