"""TEST INFRASTRUCTURE: one torchrun of a worker script at N ranks on this machine, bounded in time, that leaves
no process behind.

torchrun starts every rank in a session of its own, so neither the agent's process group nor its session
holds the ranks.  When the run has to be stopped (its time is up, or the test is interrupted) the agent
and every process below it are listed from /proc while the agent still runs; the agent gets SIGTERM first
(its handler sends SIGTERM to each rank's group) and a bounded wait, then SIGKILL goes to whatever of that
list still runs: to the group of each process that leads one, to the process alone otherwise.  Only then is
the output pipe drained, again with a time bound."""
import os
import signal
import subprocess
import sys
import time

TERM_WAIT = 30          # seconds the agent has to stop its ranks after SIGTERM
DRAIN_WAIT = 60         # seconds to drain the output once every process has been killed


def _procs():
    """{pid: (ppid, pgid, start time)} of every process /proc shows that has not exited (zombies left out)"""
    out = {}
    for d in os.listdir("/proc"):
        if not d.isdigit():
            continue
        try:
            with open("/proc/%s/stat" % d) as f:
                s = f.read()
        except OSError:
            continue
        v = s[s.rindex(")") + 2:].split()          # fields after the command name: state ppid pgrp ...
        if v[0] != "Z":
            out[int(d)] = (int(v[1]), int(v[2]), v[19])
    return out


def _tree(root):
    """{pid: (pgid, start time)} of root and every process below it"""
    procs = _procs()
    if root not in procs:
        return {}
    kids = {}
    for pid, (ppid, _, _) in procs.items():
        kids.setdefault(ppid, []).append(pid)
    out, todo = {}, [root]
    while todo:
        pid = todo.pop()
        out[pid] = procs[pid][1:]
        todo.extend(kids.get(pid, []))
    return out


def _alive(tree):
    """the processes of tree that still run (same pid and start time: not a reused pid)"""
    procs = _procs()
    return {pid: pg_st for pid, pg_st in tree.items() if pid in procs and procs[pid][1:] == pg_st}


def _kill(tree):
    own = os.getpgrp()
    for pid, (pgid, _) in _alive(tree).items():
        try:
            if pgid == pid and pgid != own:
                os.killpg(pgid, signal.SIGKILL)
            else:
                os.kill(pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
    deadline = time.time() + 10
    while _alive(tree) and time.time() < deadline:
        time.sleep(0.1)


def stop(p):
    """stops the torchrun p and every process below it; returns what p wrote"""
    tree = _tree(p.pid)
    if p.poll() is None:
        p.send_signal(signal.SIGTERM)
        try:
            p.wait(timeout=TERM_WAIT)
        except subprocess.TimeoutExpired:
            pass
    tree.update(_tree(p.pid))
    _kill(tree)
    try:
        out, _ = p.communicate(timeout=DRAIN_WAIT)
    except subprocess.TimeoutExpired:
        p.kill()
        p.stdout.close()
        p.wait(timeout=DRAIN_WAIT)
        out = ""
    return out or ""


def run(script, nproc, port, env=None, timeout=1200):
    """torchrun of `script` at nproc ranks (master 127.0.0.1:port) -> (return code, stdout + stderr).
    Past `timeout` seconds every rank is stopped and AssertionError raised with the end of the output; an
    interrupt stops every rank too before it propagates."""
    p = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                          "--nproc-per-node=%d" % nproc, "--master-addr", "127.0.0.1", "--master-port", str(port),
                          str(script)],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                         start_new_session=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        out = stop(p)
        raise AssertionError("torchrun at %d ranks still ran after %d s; every rank was stopped\n%s"
                             % (nproc, timeout, out[-3000:]))
    except BaseException:
        stop(p)
        raise
    return p.returncode, out
