"""Drop-in for the pieces of baseline/utils.py that are on the hot path."""
from distributed_rl_b200.per import PrioritizedMemory  # noqa: F401
from distributed_rl_b200.learner_common import make_optimizer as _mk


def getOptim(optimData, agent, floatV=False):
    """baseline/utils.py:78-132."""
    if floatV:
        params = [agent]
    elif isinstance(agent, tuple):
        params = [p for a in agent for p in a.parameters()]
    else:
        params = list(agent.parameters())
    return _mk(optimData, params, capturable=params[0].is_cuda if params else False)
