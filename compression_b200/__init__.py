"""compression_b200 -- H100-native (sm_90a) implementation of tensorflow/compression's data-parallel hot
path: range coding (multi-stream and legacy ops), PMF->CDF integerisation and GDN/IGDN, behind the
reference's own operator API (``gen_ops``, ``ContinuousBatchedEntropyModel``,
``LocationScaleIndexedEntropyModel``, ``GDN``).  All compute runs in hand-written CUDA kernels reached
through the C ABI of ``include/tfcb200.h``; there is no CPU fallback.
"""
from compression_b200 import _lib
from compression_b200._lib import InvalidArgumentError


def __getattr__(name):  # lazy: importing the package must not require torch / the built library
  import importlib
  modules = ("gen_ops", "functional", "math_ops", "distributions", "entropy_models", "gdn", "packed_tensors",
             "signal_conv", "models", "sharding", "run_length_models", "soft_round_layers", "layers", "ops", "parameters", "y4m_dataset", "image")
  if name in modules:
    return importlib.import_module("compression_b200." + name)
  exported = {
      "GDN": "gdn", "GDNParameter": "gdn", "Parameter": "parameters", "Y4MDataset": "y4m_dataset",
      "ContinuousBatchedEntropyModel": "entropy_models", "ContinuousIndexedEntropyModel": "entropy_models",
      "LocationScaleIndexedEntropyModel": "entropy_models", "EntropyBottleneck": "entropy_models",
      "UniversalBatchedEntropyModel": "entropy_models", "UniversalIndexedEntropyModel": "entropy_models",
      "NoisyDeepFactorized": "distributions", "DeepFactorized": "distributions", "NoisyNormal": "distributions",
      "NoisyLaplace": "distributions", "NoisyLogistic": "distributions",
      "round_st": "math_ops", "lower_bound": "math_ops", "upper_bound": "math_ops",
      "perturb_and_apply": "math_ops", "PackedTensors": "packed_tensors",
      "soft_round_inverse": "math_ops", "soft_round_conditional_mean": "math_ops",
      "SoftRound": "soft_round_layers", "SoftRoundConditionalMean": "soft_round_layers",
      "soft_round": "math_ops",
      "UniformNoiseAdapter": "distributions", "MonotonicAdapter": "distributions", "RoundAdapter": "distributions",
      "NoisyRoundAdapter": "distributions", "NoisyRoundedNormal": "distributions",
      "NoisyRoundedDeepFactorized": "distributions", "SoftRoundAdapter": "distributions",
      "NoisySoftRoundAdapter": "distributions", "NoisySoftRoundedNormal": "distributions",
      "NoisySoftRoundedDeepFactorized": "distributions", "estimate_tails": "distributions",
      "quantization_offset": "distributions", "lower_tail": "distributions", "upper_tail": "distributions",
      "SignalConv1D": "signal_conv", "SignalConv2D": "signal_conv", "SignalConv3D": "signal_conv", "RDFTParameter": "signal_conv", "same_padding_for_kernel": "signal_conv",
      "IdentityInitializer": "signal_conv",
      "MixtureSameFamily": "distributions", "NoisyMixtureSameFamily": "distributions",
      "NoisyNormalMixture": "distributions", "NoisyLogisticMixture": "distributions", "Normal": "distributions",
      "Logistic": "distributions", "Laplace": "distributions",
      "BLS2017Model": "models", "BMSHJ2018Model": "models", "MS2020Model": "models",
      "PowerLawEntropyModel": "run_length_models", "LaplaceEntropyModel": "run_length_models",
      "create_range_encoder": "gen_ops", "create_range_decoder": "gen_ops", "entropy_encode_channel": "gen_ops",
      "entropy_encode_index": "gen_ops", "entropy_encode_finalize": "gen_ops", "entropy_decode_channel": "gen_ops",
      "entropy_decode_index": "gen_ops", "entropy_decode_finalize": "gen_ops", "pmf_to_quantized_cdf": "gen_ops",
      "range_encode": "gen_ops", "range_decode": "gen_ops", "stochastic_round": "gen_ops",
      "run_length_encode": "gen_ops", "run_length_decode": "gen_ops", "run_length_gamma_encode": "gen_ops",
      "run_length_gamma_decode": "gen_ops",
  }
  if name in exported:
    return getattr(importlib.import_module("compression_b200." + exported[name]), name)
  raise AttributeError(name)
