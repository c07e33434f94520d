"""Weight pruning during training: the reference's pruning schedules and the choice of the pruned variables.

Mirror of
  neurst/sparsity/pruning_schedule.py      PruningSchedule, ConstantSparsity, PolynomialDecay (registered under their class
                                           names and snake_case aliases), `new()` returning None at target_sparsity 0
  neurst/sparsity/pruning_optimizer.py     the variables to prune (pruning_variable_pattern / nopruning_variable_pattern) and
                                           k = round(size * (1 - sparsity)) of the mask update
  neurst/exps/trainer.py:91-93,136-140     the trainer's flags

The schedule's step is the optimizer's `iterations` after the update: the updates applied in this run, from 1, not the global
step (examples/weight_pruning/README.md: begin / end "start from 0 not the initial_global_step").  The device evaluates the same
rules (b200st_optimizer_step with a prune schedule); the methods here are their float32 restatement on the host, used to
check and to report.
"""
import re

import numpy as np


class PruningSchedule(object):
    """Specifies when to prune and the sparsity (the fraction of zeros) at each step.  `should_prune_in_step(step)`: step >=
    begin and (step <= end or end < 0) and (step - begin) % frequency == 0."""

    def __init__(self, target_sparsity=0., begin_pruning_step=0, end_pruning_step=-1, pruning_frequency=100):
        if begin_pruning_step < 0:
            raise ValueError("begin_pruning_step should be >= 0")
        if end_pruning_step != -1 and end_pruning_step < begin_pruning_step:
            raise ValueError("begin_pruning_step should be <= end_pruning_step if end_pruning_step != -1")
        if pruning_frequency <= 0:
            raise ValueError("pruning_frequency should be > 0")
        if not 0.0 <= target_sparsity < 1.0:
            raise ValueError("target_sparsity must be in range [0,1)")
        self.target_sparsity = float(target_sparsity)
        self.begin_pruning_step = int(begin_pruning_step)
        self.end_pruning_step = int(end_pruning_step)
        self.pruning_frequency = int(pruning_frequency)

    def should_prune_in_step(self, step):
        in_range = step >= self.begin_pruning_step and (step <= self.end_pruning_step or self.end_pruning_step < 0)
        return bool(in_range and (step - self.begin_pruning_step) % self.pruning_frequency == 0)

    def sparsity_in_step(self, step):
        raise NotImplementedError

    def max_sparsity(self):
        """The largest sparsity any step reaches."""
        return np.float32(self.target_sparsity)

    @classmethod
    def new(cls, args):
        """None when target_sparsity is 0: pruning is off."""
        args = dict(args)
        if float(args.get("target_sparsity", 0.0)) == 0:
            return None
        return cls(**args)


class ConstantSparsity(PruningSchedule):
    """Pruning schedule with constant sparsity throughout training."""

    def sparsity_in_step(self, step):
        return np.float32(self.target_sparsity)


class PolynomialDecay(PruningSchedule):
    """sparsity = (initial - target) * (1 - p) ** power + target, p = clip((step - begin) / (end - begin), 0, 1), in float32.
    Refuses end < 0 (as the reference) and end == begin (where the reference divides by zero)."""

    def __init__(self, initial_sparsity=0., polynomial_power=3, **kwargs):
        super(PolynomialDecay, self).__init__(**kwargs)
        if not 0.0 <= initial_sparsity < 1.0:
            raise ValueError("initial_sparsity must be in range [0,1)")
        if self.end_pruning_step < 0:
            raise ValueError("end_pruning_step must > 0 when using PolynomialDecay.")
        if self.end_pruning_step == self.begin_pruning_step:
            raise ValueError("PolynomialDecay needs end_pruning_step > begin_pruning_step (the decay divides by their difference)")
        self.initial_sparsity = float(initial_sparsity)
        self.polynomial_power = float(polynomial_power)

    def sparsity_in_step(self, step):
        f = np.float32
        p = f(step - self.begin_pruning_step) / f(self.end_pruning_step - self.begin_pruning_step)
        p = min(f(1.0), max(f(0.0), p))
        # (initial - target) is a difference of Python floats (double), cast to float32 where it meets the float32 tensor
        return f(self.initial_sparsity - self.target_sparsity) * f(np.power(f(1.0) - p, f(self.polynomial_power))) \
            + f(self.target_sparsity)

    def max_sparsity(self):
        return np.float32(max(self.initial_sparsity, self.target_sparsity))


SCHEDULES = {"constantsparsity": ConstantSparsity, "polynomialdecay": PolynomialDecay}
SCHEDULE_FLAGS = ("initial_sparsity", "target_sparsity", "begin_pruning_step", "end_pruning_step", "pruning_frequency",
                  "polynomial_power")


def schedule_class(name):
    """ConstantSparsity / constant_sparsity, PolynomialDecay / polynomial_decay."""
    cls = SCHEDULES.get(str(name).lower().replace("_", ""))
    if cls is None:
        raise ValueError("pruning_schedule %r is unknown (ConstantSparsity, PolynomialDecay)" % name)
    return cls


def build_schedule(name, params):
    """The schedule of class `name` with `params`, or None when target_sparsity is 0 (PruningSchedule.new)."""
    cls = schedule_class(name)
    allowed = ("target_sparsity", "begin_pruning_step", "end_pruning_step", "pruning_frequency")
    if cls is PolynomialDecay:
        allowed += ("initial_sparsity", "polynomial_power")
    unknown = sorted(set(params) - set(allowed))
    if unknown:
        raise ValueError("%s does not take %s" % (cls.__name__, ", ".join(unknown)))
    return cls.new(params)


def k_of(size, sparsity):
    """Weights a turn keeps in a tensor of `size` elements: round(size * (1 - sparsity)) in float32, half to even."""
    f = np.float32
    return int(np.rint(f(size) * (f(1.0) - f(sparsity))))


def select_variables(names, pruning_variable_pattern=None, nopruning_variable_pattern=None):
    """The pruned subset of `names` (reference variable names), in their order: those matching pruning_variable_pattern; else
    those not matching nopruning_variable_pattern; else all (re.search, pruning_optimizer.py:48-61)."""
    if pruning_variable_pattern is not None:
        return [n for n in names if re.search(pruning_variable_pattern, n)]
    if nopruning_variable_pattern is not None:
        return [n for n in names if not re.search(nopruning_variable_pattern, n)]
    return list(names)


def pruned_parameters(table, pruning_variable_pattern=None, nopruning_variable_pattern=None):
    """Our parameter names (of a runtime's table) whose reference variable names (checkpoints.tf_variable_names) are pruned."""
    from neurst_b200.checkpoints import tf_variable_names
    tf_names = tf_variable_names(table)
    chosen = set(select_variables([tf_names[k] for k in table], pruning_variable_pattern, nopruning_variable_pattern))
    return [k for k in table if tf_names[k] in chosen]
