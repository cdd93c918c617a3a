from .etrainer import BaseEnsembleTrainer, EnsembleTrainer
from .gptrainer import GPTrainer, dklGPTrainer
from .trainer import BaseTrainer, ImSpecTrainer, RegTrainer, SegTrainer, clsTrainer

__all__ = ["BaseTrainer", "SegTrainer", "ImSpecTrainer", "RegTrainer", "clsTrainer", "GPTrainer", "dklGPTrainer",
           "BaseEnsembleTrainer", "EnsembleTrainer"]
