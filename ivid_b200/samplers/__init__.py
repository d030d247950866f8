from .samplers import DdpmSampler, DdimSampler, DpmSolverSampler, UniPcSampler
