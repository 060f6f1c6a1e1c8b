"""Model registry with the reference's surface (video_prediction/models/__init__.py:12-25):
`get_model_class('savp')` / `get_model_class('SAVPVideoPredictionModel')`; unknown names raise
ValueError('Invalid model %s').  Only the SAVP path is built on H100 (SURVEY.md section 8); the other
reference model families are registered so that the lookup behaves the same, but raise
NotImplementedError when requested."""
from .base_model import BaseVideoPredictionModel, VideoPredictionModel
from .savp_model import SAVPVideoPredictionModel

_OUT_OF_SCOPE = {
    'ground_truth': 'GroundTruthVideoPredictionModel',
    'repeat': 'RepeatVideoPredictionModel',
    'sna': 'SNAVideoPredictionModel',
    'dna': 'DNAVideoPredictionModel',
    'sv2p': 'SV2PVideoPredictionModel',
}


def get_model_class(model):
    model_mappings = {'savp': 'SAVPVideoPredictionModel'}
    model_mappings.update(_OUT_OF_SCOPE)
    model_class = model_mappings.get(model, model)
    if model_class == 'SAVPVideoPredictionModel':
        return SAVPVideoPredictionModel
    if model_class in _OUT_OF_SCOPE.values():
        raise NotImplementedError('%s is outside the H100 hot path (only the SAVP path is built)' % model_class)
    raise ValueError('Invalid model %s' % model)
