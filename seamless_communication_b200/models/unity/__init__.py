from ..fp8_weights import dequantize_decoder_weights
from .model import UnitYModel, UnitYNART2UModel, UnitYT2UModel, load_unity_model
from .unit_tokenizer import UnitTokenDecoder, UnitTokenEncoder, UnitTokenizer
