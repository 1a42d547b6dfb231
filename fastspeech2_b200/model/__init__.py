"""Mirror of the reference's `model` package surface (model/__init__.py): utils/model.py:8 imports
FastSpeech2 and ScheduledOptim from it, train.py:13 also FastSpeech2Loss."""
from .fastspeech2 import FastSpeech2, VoiceBank
from .training_stubs import FastSpeech2Loss, ScheduledOptim

__all__ = ["FastSpeech2", "FastSpeech2Loss", "ScheduledOptim", "VoiceBank"]
