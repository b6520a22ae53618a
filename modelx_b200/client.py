"""Python face of the C++ host mirror (include/modelx_client.h): the digest path of
``pkg/client.Client.{Push,Pull}``, ``pkg/types`` JSON and the local FS store of ``pkg/registry``.
All logic lives in modelx_b200/csrc/host/client_host.cpp; this module only marshals arguments."""
from __future__ import annotations

import ctypes as C
import json
import os
from typing import Optional

from . import _native as N
from .engine import Engine

PUSH_TREE = 1
PUSH_CACHE = 2
PUSH_FORCE_MULTIPART = 4


def _take(lib, p: C.c_void_p) -> str:
    try:
        return C.cast(p, C.c_char_p).value.decode()
    finally:
        lib.mxc_free(p)


def parse_manifest_json(basedir: str, configfile: str = "modelx.yaml", lib=None) -> str:
    """ParseManifest (pkg/client/push.go:67-100) -> the exact JSON Go's encoding/json would emit."""
    lib = lib or N.load()
    out = C.c_void_p()
    N.check(lib.mxc_parse_manifest(basedir.encode(), configfile.encode(), C.byref(out)), "mxc_parse_manifest", lib)
    return _take(lib, out)


def blob_digest_path(repository: str, digest: str, lib=None) -> str:
    lib = lib or N.load()
    out = C.c_void_p()
    N.check(lib.mxc_blob_digest_path(repository.encode(), digest.encode(), C.byref(out)), "mxc_blob_digest_path", lib)
    return _take(lib, out)


def untgz(archive: str, intodir: str, lib=None) -> None:
    """UnTGZ (pkg/client/helper.go:55-83)."""
    lib = lib or N.load()
    N.check(lib.mxc_untgz(archive.encode(), intodir.encode()), "mxc_untgz", lib)


def _tree_identity(desc: dict):
    """The modelx.tree.v1 root ("sha256:<hex>") and tree parameters of a manifest descriptor, in either form
    client_host.cpp writes: tree-keyed (``digest`` is the root, annotation ``modelx.digest = "tree.v1;leaf=..."``) or
    whole-file keyed with a tree annotation (``modelx.tree.v1 = "sha256:<root>;leaf=..."``)."""
    ann = desc.get("annotations") or {}
    if str(ann.get("modelx.digest", "")).startswith("tree.v1;"):
        root, fields = desc.get("digest"), ann["modelx.digest"].split(";")[1:]
    elif "modelx.tree.v1" in ann:
        root, *fields = str(ann["modelx.tree.v1"]).split(";")
    else:
        raise ValueError(f"blob {desc.get('name')!r} has no modelx.tree.v1 identity, only a whole-file SHA-256, which is "
                         "one serial chain the GPU cannot verify fast: push it with --tree")
    kv = dict(f.split("=", 1) for f in fields if "=" in f)
    try:
        params = {k: int(kv[k]) for k in ("chunk", "leaf", "fanout")}
    except (KeyError, ValueError):
        raise ValueError(f"blob {desc.get('name')!r}: malformed tree parameters {';'.join(fields)!r}") from None
    return root, params


class LocalRegistry:
    """FSRegistryStore over LocalFSProvider (pkg/registry/store_fs.go, fs_local.go): files on disk only."""

    def __init__(self, basepath: str, engine: Optional[Engine] = None):
        self.basepath = basepath
        self.engine = engine
        self._lib = engine._lib if engine is not None else N.load()

    def _check(self, rc, where):
        N.check(rc, where, self._lib)

    def put_blob(self, repository: str, digest: str, srcfile: str, content_type: str = "application/octet-stream",
                 verify=False) -> None:
        """verify: False/0 (reference behaviour: store unverified), True/1 (whole-file digest), "tree"/2 (tree root)."""
        ctx = self.engine.handle if self.engine else None
        mode = 2 if verify in ("tree", 2) else (1 if verify else 0)
        self._check(self._lib.mxc_fs_put_blob(ctx, self.basepath.encode(), repository.encode(), digest.encode(),
                                              content_type.encode(), srcfile.encode(), mode), "mxc_fs_put_blob")

    def exists_blob(self, repository: str, digest: str) -> bool:
        rc = self._lib.mxc_fs_exists_blob(self.basepath.encode(), repository.encode(), digest.encode())
        if rc < 0:
            raise N.MxdError(rc, "mxc_fs_exists_blob", self._lib)
        return bool(rc)

    def put_manifest(self, repository: str, reference: str, manifest_json: str,
                     content_type: str = "application/vnd.modelx.model.manifest.v1.json") -> None:
        self._check(self._lib.mxc_fs_put_manifest(self.basepath.encode(), repository.encode(), reference.encode(),
                                                  content_type.encode(), manifest_json.encode()), "mxc_fs_put_manifest")

    def get_manifest_json(self, repository: str, reference: str) -> str:
        out = C.c_void_p()
        self._check(self._lib.mxc_fs_get_manifest(self.basepath.encode(), repository.encode(), reference.encode(),
                                                  C.byref(out)), "mxc_fs_get_manifest")
        return _take(self._lib, out)

    def get_index(self, repository: str = "") -> dict:
        """types.Index of a repository (its pushed versions) or, with no repository, of the whole registry."""
        out = C.c_void_p()
        self._check(self._lib.mxc_fs_get_index(self.basepath.encode(), repository.encode() if repository else None,
                                               C.byref(out)), "mxc_fs_get_index")
        return json.loads(_take(self._lib, out))


class Client:
    """The digest path of pkg/client.Client (push.go / pull.go) on a GPU engine."""

    def __init__(self, engine: Engine):
        self.engine = engine
        self._lib = engine._lib

    def _check(self, rc, where):
        N.check(rc, where, self._lib)

    def push_digest_json(self, basedir: str, configfile: str = "modelx.yaml", with_tree: bool = False,
                         use_cache: bool = False) -> str:
        out = C.c_void_p()
        flags = (PUSH_TREE if with_tree else 0) | (PUSH_CACHE if use_cache else 0)
        self._check(self._lib.mxc_push_digest(self.engine.handle, basedir.encode(), configfile.encode(),
                                              flags, C.byref(out)), "mxc_push_digest")
        return _take(self._lib, out)

    def tgz(self, directory: str, intofile: Optional[str] = None):
        """TGZ (helper.go:24-53) -> (digest string, archive bytes)."""
        out = C.c_void_p()
        size = C.c_uint64()
        self._check(self._lib.mxc_tgz(self.engine.handle, directory.encode(), intofile.encode() if intofile else None,
                                      C.byref(out), C.byref(size)), "mxc_tgz")
        return _take(self._lib, out), size.value

    def pull_check(self, basedir: str, manifest_json: str) -> list:
        out = C.c_void_p()
        self._check(self._lib.mxc_pull_check(self.engine.handle, basedir.encode(), manifest_json.encode(), C.byref(out)),
                    "mxc_pull_check")
        return json.loads(_take(self._lib, out))

    @staticmethod
    def _report(text: str) -> dict:
        rep = json.loads(text)
        rep["manifest_json"] = text[len('{"manifest":'):text.rindex(',"blobs":[')]
        return rep

    def push(self, registry: LocalRegistry, repository: str, version: str, basedir: str,
             configfile: str = "modelx.yaml", force_multipart: bool = False) -> dict:
        """Client.Push (push.go:29-65) against the in-process FS store; every blob is read from disk once."""
        out = C.c_void_p()
        self._check(self._lib.mxc_push_local(self.engine.handle, basedir.encode(), configfile.encode(),
                                             registry.basepath.encode(), repository.encode(), version.encode(),
                                             PUSH_FORCE_MULTIPART if force_multipart else 0, C.byref(out)), "mxc_push_local")
        return self._report(_take(self._lib, out))

    def push_stream(self, basedir: str, uploader, configfile: str = "modelx.yaml", force_multipart: bool = False,
                    max_concurrent: int = 0) -> dict:
        """Read-once push into a part uploader (S3Extension.Upload's role).  ``uploader`` is an object with
        ``begin(blob, name, size, parts)``, ``part_write(blob, part, offset, data) -> bool``,
        ``complete(blob, digest, part_digests) -> "done"|"exists"|"empty"`` and optionally ``part_restart(blob, part)``
        and ``abort(blob)``."""
        def _begin(user, blob, name, size, parts, nparts):
            try:
                uploader.begin(blob, name.decode(), size, [(parts[i].offset, parts[i].length) for i in range(nparts)])
                return 0
            except Exception:
                return 1

        def _write(user, blob, part, offset, data, n):
            try:
                return 0 if uploader.part_write(blob, part, offset, C.string_at(data, n)) is not False else 1
            except Exception:
                return 1

        def _restart(user, blob, part):
            try:
                if hasattr(uploader, "part_restart"):
                    uploader.part_restart(blob, part)
                return 0
            except Exception:
                return 1

        def _complete(user, blob, digest, pd, nparts, status):
            try:
                raw = C.string_at(pd, 32 * nparts)
                st = uploader.complete(blob, digest.decode(), [raw[32 * i:32 * i + 32] for i in range(nparts)]) or "done"
                C.memmove(status, st.encode()[:15] + b"\0", min(len(st), 15) + 1)
                return 0
            except Exception:
                return 1

        def _abort(user, blob):
            if hasattr(uploader, "abort"):
                uploader.abort(blob)

        up = N.Uploader(None, max_concurrent, N.UP_BEGIN(_begin), N.UP_PART_WRITE(_write), N.UP_PART_RESTART(_restart),
                        N.UP_COMPLETE(_complete), N.UP_ABORT(_abort))
        out = C.c_void_p()
        self._check(self._lib.mxc_push_stream(self.engine.handle, basedir.encode(), configfile.encode(), C.byref(up),
                                              PUSH_FORCE_MULTIPART if force_multipart else 0, C.byref(out)), "mxc_push_stream")
        return self._report(_take(self._lib, out))

    def push_tree(self, registry: LocalRegistry, repository: str, version: str, basedir: str,
                  configfile: str = "modelx.yaml") -> dict:
        """Read-once, tree-keyed push (SURVEY 8f.1): each blob streams once through the pinned ring to the GPU
        (modelx.tree.v1) and into the store, and is stored under its tree root."""
        out = C.c_void_p()
        self._check(self._lib.mxc_push_local_tree(self.engine.handle, basedir.encode(), configfile.encode(),
                                                  registry.basepath.encode(), repository.encode(), version.encode(),
                                                  C.byref(out)), "mxc_push_local_tree")
        return self._report(_take(self._lib, out))

    def load_safetensors(self, registry: LocalRegistry, repository: str, version: str, name: str, device=None) -> dict:
        """Load the ``.safetensors`` blob `name` of a pushed version straight from the store into CUDA tensors on
        `device`, verified against the tree root its manifest carries (checkpoint.load_safetensors): the blob is read
        once, and no copy of it is written.  -> {tensor name: tensor}; DigestMismatch when the stored bytes are not
        the pushed ones."""
        from .checkpoint import load_safetensors
        manifest = json.loads(registry.get_manifest_json(repository, version))
        descs = [d for d in manifest.get("blobs") or [] if d.get("name") == name]
        if not descs:
            raise ValueError(f"{repository}:{version} has no blob named {name!r}")
        desc = descs[0]
        root, params = _tree_identity(desc)
        path = os.path.join(registry.basepath, blob_digest_path(repository, desc["digest"], self._lib))
        tensors, _, _, _ = load_safetensors(self.engine, path, device, expect=root, **params)
        return tensors

    def pull(self, registry: LocalRegistry, repository: str, version: str, into: str) -> list:
        """Client.Pull (pull.go:19-39) against the in-process FS store; copies are verified while they are written."""
        out = C.c_void_p()
        self._check(self._lib.mxc_pull_local(self.engine.handle, registry.basepath.encode(), repository.encode(),
                                             version.encode(), into.encode(), C.byref(out)), "mxc_pull_local")
        return json.loads(_take(self._lib, out))
