"""Python restatement of DDMin with RandomScheduler as the TestOracle (RunnerUtils.randomDDMin, RunnerUtils.scala:
601-623), on top of the Execution restatement in micro_oracle.py.  A test is RandomScheduler.test(subsequence)
(RandomScheduler.scala:597-612) over explore (:234-272): up to N executions, returning at the first that finds the
violation; execution j runs FullyRandom(seed + j).  MinimizationStats counts executions: explore increments
total_replays once per execution (:251-253) and record_iteration_size keys by total_replays (Minimizer.scala:183-185).

ORACLE — test infrastructure only.  Shares no code with oracle/random_ddmin.c."""
import micro_oracle as M


def random_test(run_one, n_execs, seed_base):
    """explore: run_one(seed) -> violation code or 0.  (first_hit, executions_run, violation)."""
    for j in range(n_execs):
        v = run_one(seed_base + j)
        if v:
            return j, j + 1, v
    return -1, n_execs, 0


class RandomDDMin(object):
    """DDMin.minimize / ddmin2 (DeltaDebugging.scala:27-109) with test(events) -> (first_hit, executions_run, violation).
    Records the sequential walk: the tested index sets, their records, and the keyed iteration-size series."""

    def __init__(self, test):
        self.test = test

    def minimize(self, events, check_unmodified=False):
        dag = list(enumerate(events))
        if check_unmodified and self.test(events)[0] < 0:                  # :41-47
            raise ValueError("Unmodified trace does not trigger violation")
        self.original, self.pruned, self.total_replays = len(dag), 0, 0   # _stats.reset() (:48)
        self.tests, self.records, self.sizes, self.keys = [], [], [], []
        mcs = self.ddmin2(dag, [])
        assert self.original - self.pruned == len(mcs)                     # :58
        self.sizes.append(self.original - self.pruned)                     # fencepost :60
        self.keys.append(self.total_replays)
        return [i for i, _ in mcs]

    def ddmin2(self, dag, remainder):
        atoms = M.atomic_events(dag)
        if len(atoms) <= 1:                                                # :74-77
            return dag
        keep = M.split_list(atoms, 2)
        for chunk in keep:                                                 # left half, then right half (:82-102)
            split = sorted(x for a in chunk for x in a)
            union = sorted(set(split) | set(remainder))
            rec = self.test([e for _, e in union])
            self.tests.append(tuple(i for i, _ in union))
            self.records.append(rec)
            self.total_replays += rec[1]                                   # one increment_replays per execution
            self.sizes.append(self.original - self.pruned)                 # record_iteration_size (:97)
            self.keys.append(self.total_replays)
            if rec[0] >= 0:
                self.pruned += len(dag) - len(split)
                return self.ddmin2(split, remainder)
        s0 = sorted(x for a in keep[0] for x in a)
        s1 = sorted(x for a in keep[1] for x in a)
        left = self.ddmin2(s0, sorted(set(s1) | set(remainder)))           # interference :104-108
        right = self.ddmin2(s1, sorted(set(s0) | set(remainder)))
        return sorted(set(left) | set(right))


def random_ddmin(run_one, events, n_execs, seed_base, check_unmodified=False):
    """run_one(subsequence, seed) -> violation code or 0.  Returns (RandomDDMin, MCS indices, verified)."""
    d = RandomDDMin(lambda sub: random_test(lambda s: run_one(sub, s), n_execs, seed_base))
    mcs = d.minimize(events, check_unmodified)
    verified = True
    if len(mcs) < len(events):                                             # verify_mcs (RunnerUtils.scala:612-620)
        verified = random_test(lambda s: run_one([events[i] for i in mcs], s), n_execs, seed_base)[0] >= 0
    return d, mcs, verified
