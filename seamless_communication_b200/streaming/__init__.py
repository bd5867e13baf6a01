from .batch import StreamingS2STBatch
from .text_decoder_policy import MMATextDecoderPolicy
