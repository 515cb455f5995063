"""ktransformers_b200 — H100-native (sm_90a) drop-in for kt-kernel's quantized-MoE decode hot path.

Layout mirrors the slice of the reference it replaces:

    native.py                ctypes face of libktb200.so (the C-ABI in include/ktb200.h); the product
                             path FAILS LOUDLY when that library is missing — there is no CPU fallback.
    util/custom_gguf.py      GGUF constants, name translation   (archive/ktransformers/util/custom_gguf.py)
    util/custom_loader.py    GGUFLoader                          (archive/ktransformers/util/custom_loader.py)
    util/utils.py            InferenceState, load_weights, ...   (archive/ktransformers/util/utils.py)
    operators/               BaseInjectedModule, KExperts*, KLinear*, KMoEGate, KDeepseekV3MoE
    optimize/                gen_optimize_config / inject / optimize_and_load_gguf + YAML rules
    models/                  the minimal DeepSeek MoE block definitions the rules match against
"""
__version__ = "0.1.0"
