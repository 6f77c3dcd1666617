"""lm:// wire headers -- byte-compatible with lmcache/protocol.py:4-70 so the reference's
`python -m lmcache.server` and this package's client/server interoperate.

client -> server: struct "ii150s" = (command, payload length, key padded to 150 bytes)  (158 bytes)
server -> client: struct "ii"     = (status code, payload length)                        (8 bytes)

This project's servers also answer three ranged-read commands (OPEN / READ / CLOSE, see csrc/lmnet.cu).  The reference
server ignores a command it does not know: it sends no reply and reads whatever body follows as the next header, so a
client that sent one would wait forever.  A client therefore sends them only after EXIST on RANGES_PROBE_KEY answered
SUCCESS (the reference answers FAIL).
"""
import struct
from dataclasses import dataclass

MAX_KEY_LENGTH = 150
_CLIENT_FMT = f"ii{MAX_KEY_LENGTH}s"
_SERVER_FMT = "ii"
RANGES_PROBE_KEY = "b200kv-ranges-v1"   # EXIST on it: SUCCESS from a server that has OPEN / READ / CLOSE
MAX_HANDLES = 4096                      # open handles a server keeps per connection
MAX_REPLY = (1 << 31) - 1               # a reply's length is an int32
OPEN_META = struct.Struct("<IIQ")       # OPEN reply: handle, 0, value size
READ_ENTRY = struct.Struct("<IIQQ")     # READ entry: handle, 0, offset, nbytes


class Constants:
    CLIENT_PUT = 1
    CLIENT_GET = 2
    CLIENT_EXIST = 3
    CLIENT_LIST = 4
    CLIENT_OPEN = 5      # key, length = prefix bytes -> u32 handle, u32 0, u64 size, then min(prefix, size) bytes
    CLIENT_READ = 6      # length = 24 m: m x (u32 handle, u32 0, u64 offset, u64 nbytes) -> the ranges in order
    CLIENT_CLOSE = 7     # length = 4 m: m x u32 handle

    SERVER_SUCCESS = 200
    SERVER_FAIL = 400


@dataclass
class ClientMetaMessage:
    command: int
    key: str
    length: int

    def serialize(self) -> bytes:
        assert len(self.key) <= MAX_KEY_LENGTH, f"Key length {len(self.key)} exceeds maximum {MAX_KEY_LENGTH}"
        return struct.pack(_CLIENT_FMT, self.command, self.length, self.key.encode().ljust(MAX_KEY_LENGTH))

    @staticmethod
    def deserialize(s: bytes) -> "ClientMetaMessage":
        command, length, key = struct.unpack(_CLIENT_FMT, s)
        return ClientMetaMessage(command, key.decode().strip(), length)

    @staticmethod
    def packlength() -> int:
        return struct.calcsize(_CLIENT_FMT)


@dataclass
class ServerMetaMessage:
    code: int
    length: int

    def serialize(self) -> bytes:
        return struct.pack(_SERVER_FMT, self.code, self.length)

    @staticmethod
    def packlength() -> int:
        return struct.calcsize(_SERVER_FMT)

    @staticmethod
    def deserialize(s: bytes) -> "ServerMetaMessage":
        code, length = struct.unpack(_SERVER_FMT, s)
        return ServerMetaMessage(code, length)
