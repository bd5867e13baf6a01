from .unit_extractor import KMEANS_10K_SHAPE, UnitExtractor
