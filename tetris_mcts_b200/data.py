"""The reference's on-disk trajectory row (SURVEY §8f.3): util/Data.py:14-26 `State(tables.IsDescription)` and its writer
DataSaver.add / add_raw / close (util/Data.py:42-132), for batched self-play.

The row is reproduced as a numpy structured dtype with PyTables' on-disk field order (an IsDescription without explicit positions is laid
out alphabetically) and the same column dtypes / shapes, so a `tables.Table.append(rows)` takes the arrays as they are.  PyTables / HDF5
are NOT installed in this image (no `tables`, no `h5py`): when `tables` is importable the saver writes the reference's HDF5 table
(`/State`, file name save_dir + save_file + str(cycle), util/Data.py:46-58); otherwise it writes the same rows as `<file>.npy` chunks
(numpy structured arrays of STATE_DTYPE) and says so.  tools/plot_*.py / replay.py read HDF5, so only the first form is byte-compatible."""
import os

import numpy as np

n_actions = 7

# util/Data.py:14-26, in PyTables' alphabetical column order
STATE_DTYPE = np.dtype([("action", np.int8), ("board", np.int8, (20, 10)), ("child_stats", np.float32, (3, n_actions)), ("combo", np.int32),
                        ("cycle", np.int32), ("episode", np.int32), ("line_stats", np.int32, (4,)), ("lines", np.int32),
                        ("policy", np.float32, (n_actions,)), ("score", np.int32), ("value", np.float32), ("variance", np.float32)])


def have_pytables():
    try:
        import tables  # noqa: F401
        return True
    except Exception:
        return False


def state_description():
    """The reference's `State` description built at run time (needs PyTables)."""
    import tables

    class State(tables.IsDescription):              # util/Data.py:14-26, column for column
        episode = tables.Int32Col()
        board = tables.Int8Col(shape=(20, 10))
        policy = tables.Float32Col(shape=(n_actions,))
        action = tables.Int8Col()
        combo = tables.Int32Col()
        lines = tables.Int32Col()
        line_stats = tables.Int32Col(shape=(4,))
        score = tables.Int32Col()
        child_stats = tables.Float32Col(shape=(3, n_actions))
        cycle = tables.Int32Col()
        value = tables.Float32Col()
        variance = tables.Float32Col()
    return State


def rows_from_batch(episode, boards, policy, action, combo, lines, line_stats, score, child_stats, cycle, value, variance):
    """One row per game of a batched move (DataSaver.add_raw, util/Data.py:98-122, vectorised)."""
    n = len(action)
    r = np.zeros(n, STATE_DTYPE)
    r["episode"], r["board"], r["policy"], r["action"] = episode, np.asarray(boards, np.int8).reshape(n, 20, 10), policy, action
    r["combo"], r["lines"], r["line_stats"], r["score"] = combo, lines, line_stats, score
    r["child_stats"], r["cycle"], r["value"], r["variance"] = child_stats, cycle, value, variance
    return r


def rows_from_move(recs_before, actions, stats, cycle, episodes, value=None, variance=None):
    """The rows play.py:131-132 saves (saver.add(ngames, action, agent, game) BEFORE game.play) for every game of a batched move:
    recs_before = the packed games the search ran on, stats = stats[n,3,7] of compute_stats (agents/agent.py:153-179), policy =
    get_prob() = visits / sum(visits) (agents/agent.py:187-189).  value / variance default to 0 when not supplied (util/Data.py:87-88)."""
    from . import pyTetris as PT
    recs = np.ascontiguousarray(recs_before, np.uint32).reshape(-1, 20)
    n = len(recs)
    stats = np.asarray(stats, np.float32).reshape(n, 3, n_actions)
    tot = stats[:, 0].sum(axis=1, keepdims=True)
    policy = np.divide(stats[:, 0], tot, out=np.zeros_like(stats[:, 0]), where=tot > 0)
    return rows_from_batch(np.asarray(episodes, np.int32), PT.states_of(recs), policy, np.asarray(actions, np.int8),
                           (recs[:, 11] >> 8).astype(np.int32), recs[:, 14].astype(np.int32), recs[:, 15:19].astype(np.int32),
                           recs[:, 13].astype(np.int32), stats, np.int32(cycle), 0 if value is None else value, 0 if variance is None else variance)


class DataSaver:
    """util/Data.py:42-132 for batched rows: add_rows(rows) appends, flushing every `chunksize` rows; close() flushes and closes."""

    def __init__(self, save_dir, save_file, cycle, chunksize=500, suffix=""):
        self.file_name = save_dir + save_file + str(cycle) + suffix  # util/Data.py:46; suffix: one file per rank of a multi-GPU run
        self.chunksize, self.cycle, self.pending, self.n_rows = chunksize, cycle, [], 0
        self.hdf5 = have_pytables()
        if self.hdf5:
            import tables
            self.file = tables.open_file(self.file_name, mode='a')
            self.table = self.file.root.State if self.file.__contains__('/State') else self.file.create_table(self.file.root, 'State', state_description())
        else:
            self.file, self.table, self.chunk = None, None, 0
            os.makedirs(os.path.dirname(self.file_name) or ".", exist_ok=True)

    def add_rows(self, rows):
        rows = np.asarray(rows, STATE_DTYPE)
        self.pending.append(rows)
        self.n_rows += len(rows)
        if sum(len(p) for p in self.pending) >= self.chunksize:
            self.flush()

    def flush(self):
        if not self.pending:
            return
        rows = np.concatenate(self.pending)
        self.pending = []
        if self.hdf5:
            self.table.append(rows)
            self.table.flush()
        else:
            np.save("%s.%06d.npy" % (self.file_name, self.chunk), rows)
            self.chunk += 1

    def close(self):                                                # util/Data.py:124-128
        self.flush()
        if self.hdf5:
            self.file.close()
