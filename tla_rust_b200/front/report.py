"""TLC-format reporting: error traces, final statistics (format pinned by
README.md:267-321 and AdvancedExamples/testout2:1-10,257-267)."""
from __future__ import annotations

from .values import fmt

OK, INVARIANT, ASSERT, DEADLOCK, EVAL_ERROR, PROPERTY = "ok", "invariant", "assert", "deadlock", "eval_error", "property"
LIVENESS = "liveness"


class CheckResult:
    def __init__(self):
        self.verdict = OK
        self.generated = 0
        self.distinct = 0
        self.queue = 0
        self.depth = 0
        self.init_states = 0
        self.trace = []          # list of (state dict, action label or None)
        self.error_text = None   # assert message / invariant name / eval error
        self.error_positions = []  # nested expression positions (assert)
        self.invariant = None
        self.levels = []         # distinct states discovered per level (for parity debugging)
        self.seconds = 0.0
        self.extra = {}
        self.back_to = None      # LIVENESS: (1-based state the cycle goes back to, action label) or None: stuttering

    def summary(self):
        return dict(verdict=self.verdict, generated=self.generated, distinct=self.distinct,
                    queue=self.queue, depth=self.depth, init=self.init_states)


def action_label(act, module):
    if act is None:
        return "<Initial predicate>"
    if isinstance(act, str):
        return act
    _, name, (l, c, el, ec), mod = act
    return f"<Action line {l}, col {c} to line {el}, col {ec} of module {mod}>"


def format_state(state: dict, var_order):
    return "\n".join(f"/\\ {v} = {fmt(state[v])}" for v in var_order)


def format_trace(res: CheckResult, var_order, module):
    out = ["Error: The behavior up to this point is:"]
    for i, (st, act) in enumerate(res.trace, 1):
        out.append(f"State {i}: {action_label(act, module)}")
        out.append(format_state(st, var_order))
        out.append("")
    return "\n".join(out)


def format_result(res: CheckResult, var_order, module):
    out = []
    if res.verdict == OK:
        out.append("Model checking completed. No error has been found.")
        out.append("  Estimates of the probability that TLC did not check all reachable states")
        out.append("  because two distinct states had the same fingerprint:")
        n = res.distinct
        p = (n * max(res.generated - n, 0)) / 2.0 ** 64
        out.append(f"  calculated (optimistic):  val = {p:.1E}")
    else:
        if res.verdict == ASSERT:
            out.append("The first argument of Assert evaluated to FALSE; the second argument was:")
            out.append(fmt(res.error_text))
        elif res.verdict == INVARIANT:
            out.append(f"Error: Invariant {res.invariant} is violated.")
        elif res.verdict == DEADLOCK:
            out.append("Error: Deadlock reached.")
        elif res.verdict == LIVENESS:
            out.append("Error: Temporal properties were violated.")
            out.append("")
            out.append("Error: The following behavior constitutes a counter-example:")
            out.append("")
            for i, (st, act) in enumerate(res.trace, 1):
                out.append(f"State {i}: {action_label(act, module)}")
                out.append(format_state(st, var_order))
                out.append("")
            if res.back_to is None:
                out.append(f"State {len(res.trace) + 1}: Stuttering")
            else:
                out.append(f"Back to state {res.back_to[0]}: {action_label(res.back_to[1], module)}")
            out.append("")
        elif res.verdict == PROPERTY:
            out.append(f"Error: Action property {res.invariant} is violated.")
        else:
            out.append(f"Error: {res.error_text}")
        if res.verdict != LIVENESS:
            out.append(format_trace(res, var_order, module))
        if res.error_positions:
            out.append("Error: The error occurred when TLC was evaluating the nested")
            out.append("expressions at the following positions:")
            for i, (l, c, el, ec) in enumerate(res.error_positions):
                out.append(f"{i}. Line {l}, column {c} to line {el}, column {ec} in {module}")
            out.append("")
            out.append("")
    out.append(f"{res.generated} states generated, {res.distinct} distinct states found, "
               f"{res.queue} states left on queue.")
    out.append(f"The depth of the complete state graph search is {res.depth}.")
    return "\n".join(out)
