from .generator import BannedSequenceProcessor, NGramRepeatBlockProcessor, SequenceGeneratorOptions, UnitYGenerator
from .translator import BatchedSpeechOutput, Modality, Task, Translator
from .transcriber import Transcriber, Transcription, TranscriptionToken, TranscriptionTokenStats
