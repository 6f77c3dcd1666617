"""Connector factory (lmcache/storage_backend/connector/__init__.py:28-102).  Only the transport the
north-star deployment uses is provided here: `lm://host:port` (one lmcache.server over host sockets).  Both clients speak
the same wire protocol and both send from / receive into page-locked slabs without copies: `lm://` is the Python-socket
client, `lmn://` the client of the
native library (csrc/lmnet.cu).
`redis://` needs the external redis client and is outside the rebuilt hot path."""
import re

from lmcache_b200.storage_backend.connector.base_connector import RemoteConnector
from lmcache_b200.storage_backend.connector.lm_connector import LMCServerConnector
from lmcache_b200.storage_backend.connector.native_connector import LMCNativeConnector

_URL = re.compile(r"^(?P<scheme>[a-z][a-z0-9+.-]*)://(?P<host>[^:/]+):(?P<port>\d+)$")


def CreateConnector(url: str) -> RemoteConnector:
    m = _URL.match(url)
    if not m:
        raise ValueError(f"Invalid remote url: {url}")
    scheme, host, port = m.group("scheme"), m.group("host"), int(m.group("port"))
    if scheme == "lm":
        return LMCServerConnector(host, port)
    if scheme == "lmn":
        return LMCNativeConnector(host, port)
    raise ValueError(f"Unsupported connector type {scheme} (lmcache_b200 provides lm:// only)")


__all__ = ["RemoteConnector", "LMCServerConnector", "LMCNativeConnector", "CreateConnector"]
