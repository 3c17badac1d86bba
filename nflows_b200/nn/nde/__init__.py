from .made import MixtureOfGaussiansMADE
