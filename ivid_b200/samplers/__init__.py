from .samplers import DdpmSampler, DdimSampler, DpmSolverSampler, UniPcSampler, init_steps
