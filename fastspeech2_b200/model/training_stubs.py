"""Training-side names the reference's `model` package exports (model/loss.py, model/optimizer.py).

Training is outside this path's scope (SURVEY.md section 2.1 rows 11-13); the names exist so that
`from model import FastSpeech2, ScheduledOptim` (utils/model.py:8) keeps importing.  Using them raises."""


class _TrainingOnly:
    def __init__(self, *a, **k):
        raise NotImplementedError(f"{type(self).__name__}: the H100-native drop-in covers inference only")


class FastSpeech2Loss(_TrainingOnly):
    pass


class ScheduledOptim(_TrainingOnly):
    pass
