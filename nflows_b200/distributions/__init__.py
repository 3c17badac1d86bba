from .base import Distribution, NoMeanException
from .normal import ConditionalDiagonalNormal, DiagonalNormal, StandardNormal
from .mixture import MADEMoG
