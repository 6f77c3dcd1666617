"""Record the lm:// wire exchange of LMCache v0.1.2's own client and server (CPU, once):

    python tests/golden/make_lm_wire.py <path of an LMCache v0.1.2 tree>

The reference's LMCServerConnector (lmcache/storage_backend/connector/lm_connector.py:15-84) talks to the reference's
server (python -m lmcache.server, lmcache/server/__main__.py:29-104) through a recording proxy.  Output (committed):
tests/golden/golden_lm_wire.npz -- per call of the session below, the bytes the client sent (c2s_<i>) and the bytes the
server answered (s2c_<i>), plus the session itself as JSON (calls).  Every value is a run of one byte value, so the
compressed file stays small.  tests/test_c4_flow_cpu.py replays it against this package's clients and server.
"""
import json
import os
import socket
import subprocess
import sys
import threading
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = [1, 157, 65536, 2 * 1024 * 1024 + 3]      # one byte, odd lengths, more than one socket read
HDR = 158                                         # ClientMetaMessage.packlength()


def key(i):
    return "vllm@lmsys/longchat-7b-16k@2@0@" + ("f" * 64 if i < 0 else "%064x" % i)


def session():
    """(op, key index): every value is PUT, then EXIST / GET / GET of each, then a key nobody stored, then LIST"""
    calls = [("set", i) for i in range(len(SIZES))]
    for i in range(len(SIZES)):
        calls += [("exists", i), ("get", i), ("get", i)]
    return calls + [("exists", -1), ("get", -1), ("list", None)]


class Proxy:
    """one client connection forwarded to the server; both byte streams recorded"""

    def __init__(self, upstream_port):
        self.ls = socket.create_server(("127.0.0.1", 0))
        self.port = self.ls.getsockname()[1]
        self.up = upstream_port
        self.c2s, self.s2c = bytearray(), bytearray()
        threading.Thread(target=self._accept, daemon=True).start()

    def _accept(self):
        a, _ = self.ls.accept()
        b = socket.create_connection(("127.0.0.1", self.up))
        threading.Thread(target=self._pump, args=(a, b, self.c2s), daemon=True).start()
        threading.Thread(target=self._pump, args=(b, a, self.s2c), daemon=True).start()

    @staticmethod
    def _pump(src, dst, log):
        while True:
            d = src.recv(1 << 20)
            if not d:
                dst.close()
                return
            log.extend(d)          # recorded before it is forwarded: a reply the client has read is complete here
            dst.sendall(d)


def main(ref):
    sys.path[:0] = [os.path.join(HERE, "..", "_refstubs"), ref]
    from lmcache.storage_backend.connector.lm_connector import LMCServerConnector

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(HERE, "..", "_refstubs"), ref]))
    srv = subprocess.Popen([sys.executable, "-m", "lmcache.server", "127.0.0.1", str(port)], env=env,
                           stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    try:
        for _ in range(300):
            try:
                socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
                break
            except OSError:
                time.sleep(0.1)
        px = Proxy(port)
        c = LMCServerConnector("127.0.0.1", px.port)
        out, calls = {}, []
        sent = 0
        for n, (op, i) in enumerate(session()):
            c0, s0 = len(px.c2s), len(px.s2c)
            rec = {"op": op, "key": key(i) if i is not None else ""}
            if op == "set":
                rec.update(byte=i + 1, size=SIZES[i])
                c.set(rec["key"], bytes([i + 1]) * SIZES[i])
                sent += HDR + SIZES[i]
                while len(px.c2s) < sent:          # PUT has no reply: wait until the proxy has seen all of it
                    time.sleep(0.01)
            else:
                got = getattr(c, op)(rec["key"]) if op != "list" else c.list()
                sent += HDR
                rec["want"] = (list(got) if op == "list" else bool(got) if op == "exists" else
                               None if got is None else {"byte": int(got[0]), "size": len(got)})
            assert len(px.c2s) == sent
            out[f"c2s_{n}"] = np.frombuffer(bytes(px.c2s[c0:]), np.uint8)
            out[f"s2c_{n}"] = np.frombuffer(bytes(px.s2c[s0:]), np.uint8)
            calls.append(rec)
        c.close()
        out["calls"] = np.frombuffer(json.dumps(calls).encode(), np.uint8)
        np.savez_compressed(os.path.join(HERE, "golden_lm_wire.npz"), **out)
    finally:
        srv.terminate()
        srv.wait()


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
