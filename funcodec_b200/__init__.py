"""funcodec_b200: H100-native (sm_90a) codec encode -> RVQ -> decode hot path for FunCodec."""
from .config import CodecConfig, PRESETS, get_config  # noqa: F401
from .weights import init_state_dict, state_dict_shapes, conv_specs  # noqa: F401

__version__ = "0.1.0"
