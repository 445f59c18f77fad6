"""The writer thread of the evaluator and visualizer drop-ins (lib/evaluators/if_nerf.py, lib/visualizers/): cv2.imwrite and
a file's write() release the GIL, so the next view renders while one thread encodes and writes the last one's files."""
import queue
import threading


class PngWriter:
    """One daemon thread that runs jobs in order from a small bounded queue (`put` blocks while it is full).  A job is a
    (path, uint8 BGR array) pair, or `make`, a callable returning that pair, run on the thread after `event` (anything with
    a `synchronize()`, e.g. a torch.cuda.Event) has completed; a `make` that returns None has written its own file (the
    mesh visualizer's PLY).  `done` runs after the job whatever happens, also when it is skipped.  The first error (a
    job's exception, or IOError when cv2.imwrite returns False) is kept, the jobs after it are skipped, and it is raised in
    the caller's thread by the next `put`, `check` or `join`."""

    def __init__(self, depth=4, name="png-writer"):
        self._q = queue.Queue(maxsize=depth)
        self._error = None
        self._thread = None
        self._name = name

    def _run(self):
        while True:
            event, make, done = self._q.get()
            try:
                if self._error is None:
                    if event is not None:
                        event.synchronize()
                    job = make() if callable(make) else make
                    if job is not None:
                        import cv2
                        path, img = job
                        if not cv2.imwrite(path, img):
                            raise IOError("cv2.imwrite could not write %s" % path)
            except Exception as e:       # handed to the caller's thread
                self._error = e
            finally:
                try:
                    if done is not None:
                        done()
                finally:
                    self._q.task_done()

    def put(self, path, img):
        self.submit((path, img))

    def submit(self, make, event=None, done=None):
        self.check()
        if self._thread is None:
            self._thread = threading.Thread(target=self._run, name=self._name, daemon=True)
            self._thread.start()
        self._q.put((event, make, done))

    def join(self):
        self._q.join()
        self.check()

    def check(self):
        if self._error is not None:
            e, self._error = self._error, None
            raise e
