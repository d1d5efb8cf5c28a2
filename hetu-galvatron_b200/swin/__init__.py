"""The Swin family harness (``galvatron/models/swin``): the three callbacks + ModelInfo the core API asks for."""
from .meta_configs import config_from_meta, set_model_config, stage_geometry
from .SwinModel_hybrid_parallel import (construct_hybrid_parallel_model, get_hybrid_parallel_configs, get_swin_config, swin_model_hp,
                                        token_rows)
from .SwinModel_sequential import SwinModelInfo, construct_sequential_model
from .SwinModel_tensor_parallel import SwinBlock_tp, SwinDownsample_tp, construct_tensor_parallel_model, shift_mask, token_map
