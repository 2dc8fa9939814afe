"""CPU reference for the BroadcastNestedLoopJoin operator (NestedLoopJoinExec, planner.rs:1386-1436), on top of the join-condition
reference (tests/condjoinref.py), whose condition rules and resolution it keeps.  Each rule is the reference's:

- Shapes: the ones Comet's serde sends (operators.scala:2258-2266), whose output follows the streamed side:
  Inner with either build side, LeftOuter / LeftSemi / LeftAnti with BuildRight, RightOuter with BuildLeft.  The streamed side is the
  probe side: the left one unless the build side is the left one.
- There are no keys: every (left row, right row) pair is a candidate.  With a condition a pair passes when it is TRUE (bound to the left
  columns followed by the right ones); without one every pair passes.  The condition never sees a NULL-extended row.
- Order: Spark's BroadcastNestedLoopJoinExec order, streamed-row major: streamed rows in input order, each one's passing pairs in the
  other side's input order.  An outer join's streamed row with no passing pair appears once, in its place, NULL-extended.  DataFusion
  leaves the order open, so this is one of its valid answers and outputs compare bit-exact.
- Empty sides: an empty build side gives nothing for Inner and LeftSemi and every streamed row for LeftAnti and the outer types; an
  empty streamed side gives nothing."""
import condjoinref as C
from joinref import INNER, LEFT_ANTI, LEFT_SEMI
from smjref import LEFT_OUTER, RIGHT_OUTER

ACCEPTED = [(INNER, False), (INNER, True), (LEFT_OUTER, False), (RIGHT_OUTER, True), (LEFT_SEMI, False), (LEFT_ANTI, False)]


def candidates(n_left, n_right, build_left=False):
    """every (left row, right row) pair, streamed-row major"""
    if build_left:    # the right side is streamed
        return [(l, r) for r in range(n_right) for l in range(n_left)]
    return [(l, r) for l in range(n_left) for r in range(n_right)]


def output_rows(left, right, join_type, cond, build_left=False):
    """(output rows as condjoinref.resolve gives them, pairs the condition was evaluated on)"""
    if (join_type, build_left) not in ACCEPTED:
        raise ValueError(f"{join_type} nested-loop join with build_left={build_left} is not an accepted shape")
    cands = candidates(left.num_rows, right.num_rows, build_left)
    rows = C.resolve(left.num_rows, right.num_rows, cands, C.passes(left, right, cands, cond), join_type, build_left)
    return rows, candidate_count(left, right, cond)


def nlj_table(left, right, join_type, cond, build_left=False):
    """the operator's output over pa.Tables left and right"""
    rows, _ = output_rows(left, right, join_type, cond, build_left)
    return C.to_table(left, right, rows, join_type)


def candidate_count(left, right, cond):
    """the pairs the condition is evaluated on (join_cond_pairs): all of them, none when a side is empty or there is no condition"""
    return left.num_rows * right.num_rows if cond is not None else 0
