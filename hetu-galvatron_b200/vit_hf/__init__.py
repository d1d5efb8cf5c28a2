"""The ViT family harness (``galvatron/models/vit_hf``): the three callbacks + ModelInfo the core API asks for."""
from .meta_configs import config_from_meta, set_model_config
from .ViTModel_hybrid_parallel import (construct_hybrid_parallel_model, get_hybrid_parallel_configs, get_vit_config, token_rows,
                                       vit_model_hp)
from .ViTModel_sequential import ViTModelInfo, construct_sequential_model
from .ViTModel_tensor_parallel import ViTLayer_tp, construct_tensor_parallel_model
