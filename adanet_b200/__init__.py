"""adanet_b200: an H100-native AdaNet candidate-training engine behind the
tensorflow/adanet API surface (adanet/__init__.py:21-59 of the reference).

The per-iteration hot path runs as hand-written sm_90a CUDA kernels
(adanet_b200/csrc, C ABI in include/adanet_b200.h); this package is the
host-side mirror of the reference's plugin interface over it.  Importing the
package needs neither a GPU nor the built extension; any compute entry point
fails loudly without them (there is no CPU fallback).
"""

from adanet_b200 import distributed
from adanet_b200 import ensemble
from adanet_b200 import estimators
from adanet_b200 import graph
from adanet_b200 import heads
from adanet_b200 import replay
from adanet_b200 import subnetwork
from adanet_b200 import train
from adanet_b200.autoensemble import AutoEnsembleEstimator
from adanet_b200.autoensemble import AutoEnsembleSubestimator
from adanet_b200.core.estimator import Estimator
from adanet_b200.core.estimator import RunConfig
from adanet_b200.core.evaluator import Evaluator
from adanet_b200.ensemble import ComplexityRegularized
from adanet_b200.ensemble import ComplexityRegularizedEnsembler
from adanet_b200.ensemble import Ensembler
from adanet_b200.ensemble import MeanEnsemble
from adanet_b200.ensemble import MeanEnsembler
from adanet_b200.ensemble import MixtureWeightType
from adanet_b200.ensemble import WeightedSubnetwork
from adanet_b200.subnetwork import Subnetwork

# adanet/__init__.py: `adanet.Ensemble` is the ComplexityRegularized ensemble namedtuple
Ensemble = ComplexityRegularized


class Summary:
  """adanet.Summary interface (adanet/core/summary.py:40-200): what `build_subnetwork(..., summary)` receives.
  TensorBoard plumbing is outside the hot path (SURVEY.md section 8: out of scope); every call is a no-op."""

  def scalar(self, name, tensor=None, family=None, **kwargs):
    return None

  image = audio = histogram = scalar


def _out_of_scope(name, why):
  class _Unavailable:
    def __init__(self, *args, **kwargs):
      raise NotImplementedError("adanet_b200.%s is not part of the B200 engine: %s" % (name, why))
  _Unavailable.__name__ = name
  return _Unavailable


# names of the reference's top-level API that live outside the candidate-training hot path (SURVEY.md section 8:
# reports feed Generators with TF metric tensors; TPU estimators are a different accelerator's control plane)
ReportMaterializer = _out_of_scope("ReportMaterializer", "subnetwork Reports materialise TensorFlow metric ops")
TPUEstimator = _out_of_scope("TPUEstimator", "TPU control plane")
AutoEnsembleTPUEstimator = _out_of_scope("AutoEnsembleTPUEstimator", "TPU control plane")

__version__ = "0.1.0"

__all__ = [
    "AutoEnsembleEstimator", "AutoEnsembleSubestimator", "ComplexityRegularized", "ComplexityRegularizedEnsembler",
    "Ensemble", "Ensembler", "Estimator", "Evaluator", "MeanEnsemble", "MeanEnsembler", "MixtureWeightType",
    "RunConfig", "Subnetwork", "WeightedSubnetwork", "distributed", "ensemble", "estimators", "graph", "heads",
    "replay", "subnetwork", "train", "Summary", "ReportMaterializer", "TPUEstimator", "AutoEnsembleTPUEstimator",
]
