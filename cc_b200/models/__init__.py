"""Model factory with the reference's names (models/__init__.py): ``getattr(models, name)(...)``
as train.py:245-255 does.  The four architectures of the BASELINE.json path plus the reference's alternates
(SURVEY.md N4), and FlowNetC6, the second choice of --flownet (train.py:90)."""
from .DispResNet6 import DispResNet6
from .PoseNetB6 import PoseNetB6
from .MaskNet6 import MaskNet6
from .back2future import Model as Back2Future
from .alternates import DispNetS, DispNetS6, DispResNetS6, PoseNet6, PoseExpNet, MaskResNet6
from .FlowNetC6 import FlowNetC6
