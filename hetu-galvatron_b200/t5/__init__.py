"""The T5 family harness (``galvatron/models/T5``): the three callbacks + ModelInfo the core API asks for."""
from .meta_configs import config_from_meta, set_model_config
from .T5Model_hybrid_parallel import construct_hybrid_parallel_model, estimate_arena_bytes, get_hybrid_parallel_configs, get_t5_config, t5_model_hp
from .T5Model_sequential import T5ModelInfo, construct_sequential_model
from .T5Model_tensor_parallel import T5DecoderLayer_tp, T5EncoderLayer_tp, construct_tensor_parallel_model, row_index
