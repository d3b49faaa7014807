from . import flags, flops, image_transformer_v1, image_transformer_v2, image_v1
from .flags import checkpointing, get_checkpointing
from .image_transformer_v1 import ImageTransformerDenoiserModelV1
from .image_transformer_v2 import ImageTransformerDenoiserModelV2
from .image_v1 import ImageDenoiserModelV1
