"""Wire-compatible `Slave` gRPC service (SURVEY.md 8f N3): an unmodified reference `Master` JVM can drive a GPU
worker through the protocol it already speaks.

The schema is the reference's `src/main/protobuf/proto.proto` (services `Master` :13-19 and `Slave` :37-49, messages
:21-35,51-70) rebuilt at run time with protobuf descriptors -- `grpc_tools` is not installed here and the ScalaPB option
lines of the .proto (:5,8-11 and the field options) do not affect the wire format.  Every handler body is one C-ABI
call on the worker's `NativeCtx`; vectors cross the wire as `Sparse{map<int32,double>, size}` with the reference's
1-based feature keys (column c <-> key c + 1, utils/Dataset.scala:30; key == size is legal, quirk Q11).

Async mode: the reference slave forwards every delta to its colleague slaves and to the master over gRPC
(core/Slave.scala:104-105).  A GPU worker writes its deltas into GPU peers' replicas through NVLink; for colleagues that are
NOT GPU peers (slaves registered with `RegisterSlave`, a master given as `master_target`) the worker loop also adds every delta
to an OUTBOX accumulator on the device (dsgd_async_outbox_enable) and `AsyncRelay` forwards the difference since its last read
as one `UpdateGrad` message per period.  Divergence, stated: one message per period carrying the SUM of that period's deltas,
not one message per iteration -- the receivers' `w -= delta` additions commute, the master's update COUNTER however advances
by one per message, so a reference master's stop rule (`updates >= N * maxEpochs`, core/MasterAsync.scala:83,171) sees periods,
not iterations.
"""
from __future__ import annotations

import threading
from concurrent import futures
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np

PACKAGE = "epfl.distributed"


def _build_pool():
    from google.protobuf import descriptor_pb2, descriptor_pool, empty_pb2
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto()
    fd.name, fd.package, fd.syntax = "epfl_distributed_proto.proto", PACKAGE, "proto3"
    fd.dependency.append("google/protobuf/empty.proto")

    def msg(name):
        m = fd.message_type.add()
        m.name = name
        return m

    def field(m, name, number, ftype, label=F.LABEL_OPTIONAL, type_name=None, packed=None):
        f = m.field.add()
        f.name, f.number, f.type, f.label = name, number, ftype, label
        if type_name:
            f.type_name = type_name
        if packed is not None:
            f.options.packed = packed
        return f

    node = msg("Node")                                   # proto.proto:21-24
    field(node, "host", 1, F.TYPE_STRING)
    field(node, "port", 2, F.TYPE_INT32)
    msg("Ack")                                           # proto.proto:26
    sparse = msg("Sparse")                               # proto.proto:28-31
    entry = sparse.nested_type.add()
    entry.name = "MapEntry"
    entry.options.map_entry = True
    field(entry, "key", 1, F.TYPE_INT32)
    field(entry, "value", 2, F.TYPE_DOUBLE)
    field(sparse, "map", 1, F.TYPE_MESSAGE, F.LABEL_REPEATED, f".{PACKAGE}.Sparse.MapEntry")
    field(sparse, "size", 2, F.TYPE_INT32)
    gu = msg("GradUpdate")                               # proto.proto:33-35
    field(gu, "gradUpdate", 1, F.TYPE_MESSAGE, type_name=f".{PACKAGE}.Sparse")
    fr = msg("ForwardRequest")                           # proto.proto:51-54
    field(fr, "samples", 1, F.TYPE_INT32, F.LABEL_REPEATED, packed=True)
    field(fr, "weights", 2, F.TYPE_MESSAGE, type_name=f".{PACKAGE}.Sparse")
    fp = msg("ForwardReply")                             # proto.proto:56-58
    field(fp, "predictions", 1, F.TYPE_DOUBLE, F.LABEL_REPEATED)
    gr = msg("GradientRequest")                          # proto.proto:60-63
    field(gr, "weights", 1, F.TYPE_MESSAGE, type_name=f".{PACKAGE}.Sparse")
    field(gr, "samples", 2, F.TYPE_INT32, F.LABEL_REPEATED, packed=True)
    sa = msg("StartAsyncRequest")                        # proto.proto:65-70
    field(sa, "weights", 1, F.TYPE_MESSAGE, type_name=f".{PACKAGE}.Sparse")
    field(sa, "samples", 2, F.TYPE_INT32, F.LABEL_REPEATED)
    field(sa, "batchSize", 3, F.TYPE_INT32)
    field(sa, "learningRate", 4, F.TYPE_DOUBLE)

    pool = descriptor_pool.DescriptorPool()
    pool.Add(descriptor_pb2.FileDescriptorProto.FromString(empty_pb2.DESCRIPTOR.serialized_pb))
    pool.Add(fd)
    return pool


class Messages:
    """Message classes of proto.proto, built once."""
    _cache = None

    def __new__(cls):
        if cls._cache is None:
            from google.protobuf import empty_pb2, message_factory
            pool = _build_pool()
            inst = super().__new__(cls)
            for name in ("Node", "Ack", "Sparse", "GradUpdate", "ForwardRequest", "ForwardReply", "GradientRequest",
                         "StartAsyncRequest"):
                setattr(inst, name, message_factory.GetMessageClass(pool.FindMessageTypeByName(f"{PACKAGE}.{name}")))
            inst.Empty = empty_pb2.Empty
            cls._cache = inst
        return cls._cache


# ---- Vec <-> Sparse message (core/package.scala:12-13) ----------------------------------------------------------

def sparse_to_dense(sp, dim: int) -> np.ndarray:
    """`Vec(sparse.map, sparse.size)`: reference keys are 1-based feature ids; dense index = key - 1."""
    if sp.size not in (0, dim):
        raise ValueError(f"vector of size {sp.size}, expected {dim}")
    w = np.zeros(dim, dtype=np.float64)
    for k, v in sp.map.items():
        if not (1 <= k <= dim):
            raise IndexError(f"Illegal index '{k}'")          # math/Sparse.scala:62-64
        w[k - 1] = v
    return w


def dense_to_sparse(M: Messages, a: np.ndarray, dim: int):
    """`Sparse(vec.map, vec.size)`: 0.0 stands for an absent key (what the Sparse constructor filters out)."""
    sp = M.Sparse(size=dim)
    nz = np.flatnonzero(a)
    for i, v in zip(nz.tolist(), a[nz].tolist()):
        sp.map[i + 1] = v
    return sp


class AsyncRelay:
    """core/Slave.scala:104-105 for colleagues reached over the host: reads the worker's outbox (sum of -delta since it was
    enabled) every `period` seconds and sends the difference since the last read to every sender as one GradUpdate."""

    def __init__(self, ctx, dim: int, period: float = 0.05):
        self.ctx, self.dim, self.period = ctx, dim, period
        self.M = Messages()
        self.senders: Dict[object, Callable] = {}
        self.last = np.zeros(dim)
        self.sent = 0
        self.errors: List[str] = []
        self._lock = threading.Lock()
        self._stop = threading.Event()
        self._thread: Optional[threading.Thread] = None

    def add(self, key, send: Callable):
        with self._lock:
            self.senders[key] = send

    def remove(self, key):
        with self._lock:
            self.senders.pop(key, None)

    def flush(self) -> int:
        """Forwards what the worker has applied since the previous flush; returns the number of non-zero entries sent."""
        with self._lock:
            acc = self.ctx.async_outbox_read()
            diff = acc - self.last                 # = -(sum of the deltas of the period)
            self.last = acc
            nz = np.flatnonzero(diff)
            if nz.size == 0:
                return 0
            msg = self.M.GradUpdate(gradUpdate=dense_to_sparse(self.M, -diff, self.dim))   # receivers do w -= delta
            for key, send in list(self.senders.items()):
                try:
                    send(msg)
                except Exception as e:  # the reference does not await these futures either (core/Slave.scala:104-105)
                    self.errors.append(f"{key}: {type(e).__name__}: {e}")
            self.sent += 1
            return int(nz.size)

    def start(self):
        self._stop.clear()
        self._thread = threading.Thread(target=self._loop, daemon=True)
        self._thread.start()

    def _loop(self):
        while not self._stop.wait(self.period):
            self.flush()

    def stop(self):
        """Ends the periodic loop and forwards what is left (call after the worker loop has stopped)."""
        self._stop.set()
        if self._thread is not None:
            self._thread.join(timeout=5.0)
            self._thread = None
        self.flush()


class SlaveServicer:
    """Handlers of service `epfl.distributed.Slave` (proto.proto:37-49) over one device context."""

    def __init__(self, ctx, n_train: int, is_async: bool, concurrency: int = 1, seed: int = 0,
                 master_target: Optional[str] = None, relay_period: float = 0.05):
        if getattr(ctx, "intercept", False):
            # the service's Sparse weight messages are dim long: an intercept would be dropped on every request
            raise ValueError("SlaveServicer: the Slave service's weight messages carry no intercept; serve a context created "
                             "without fit_intercept")
        self.ctx, self.n_train, self.is_async = ctx, n_train, is_async
        self.dim = ctx.dim
        self.concurrency, self.seed = concurrency, seed
        self.colleagues: Dict[Tuple[str, int], bool] = {}
        self.master_target, self.relay_period = master_target, relay_period
        self.relay: Optional[AsyncRelay] = None
        self._stubs: Dict[object, object] = {}
        self.M = Messages()
        self._ctx_lock = threading.Lock()

    # registration bookkeeping (core/Slave.scala:115-127); a colleague that registers while the loop runs is sent to from the
    # next period on, like the reference's `slaves` map
    def RegisterSlave(self, node, context=None):
        self.colleagues[(node.host, node.port)] = True
        if self.relay is not None:
            self._attach((node.host, node.port))
        return self.M.Ack()

    def UnregisterSlave(self, node, context=None):
        self.colleagues.pop((node.host, node.port), None)
        if self.relay is not None:
            self.relay.remove((node.host, node.port))
        stub = self._stubs.pop((node.host, node.port), None)
        if stub is not None:
            stub.close()
        return self.M.Ack()

    def _attach(self, key):
        if key == "master":
            stub = MasterStub(self.master_target)
        else:
            stub = SlaveStub(f"{key[0]}:{key[1]}")
        self._stubs[key] = stub
        self.relay.add(key, stub.UpdateGrad)

    def _samples(self, samples) -> np.ndarray:
        idx = np.fromiter(samples, dtype=np.int64, count=len(samples))
        if idx.size and (idx.min() < 0 or idx.max() >= self.n_train):
            raise IndexError("sample id outside the training rows")   # data(idx) on the reference's array
        return idx.astype(np.int32)

    # Forward / Gradient / StartAsync share the context's request buffers (weights, gradient, counters): the C ABI wants
    # them serialised by the caller (include/dsgd.h, "Threading"), and the handlers run on a thread pool -- hence the lock.
    # UpdateGrad / StopAsync are the calls the ABI allows while the async loop runs and stay outside it.
    def Forward(self, request, context=None):             # core/Slave.scala:129-140
        idx = self._samples(request.samples)
        w = sparse_to_dense(request.weights, self.dim)
        with self._ctx_lock:
            preds = self.ctx.forward(idx, w) if idx.size else np.zeros(0)
        return self.M.ForwardReply(predictions=preds.tolist())

    def Gradient(self, request, context=None):            # core/Slave.scala:142-157
        idx = self._samples(request.samples)
        w = sparse_to_dense(request.weights, self.dim)
        with self._ctx_lock:
            grad = self.ctx.gradient(idx, w)              # empty batch -> DsgdEmpty (Vec.sum of an empty list throws)
        return self.M.GradUpdate(gradUpdate=dense_to_sparse(self.M, grad, self.dim))

    def StartAsync(self, request, context=None):          # core/Slave.scala:159-175
        if not self.is_async:
            raise RuntimeError("Cannot initialize async computation: slave is in synchronous mode.")
        idx = self._samples(request.samples)
        w = sparse_to_dense(request.weights, self.dim)
        with self._ctx_lock:
            relay = None
            if self.colleagues or self.master_target:      # somebody this worker cannot reach over NVLink
                self.ctx.async_outbox_enable()
                relay = AsyncRelay(self.ctx, self.dim, self.relay_period)
            self.ctx.start_async(w, idx, request.batchSize, request.learningRate, concurrency=self.concurrency,
                                 max_updates=0, seed=self.seed)
            if relay is not None:
                self.relay = relay
                for key in list(self.colleagues):
                    self._attach(key)
                if self.master_target:
                    self._attach("master")
                relay.start()
        return self.M.Ack()

    def StopAsync(self, request, context=None):           # core/Slave.scala:187-195
        if not self.is_async:
            raise RuntimeError("Cannot stop async computation: slave is in synchronous mode.")
        self.ctx.stop_async()
        if self.relay is not None:
            self.relay.stop()                              # forwards the rest
            self.relay = None
            for stub in self._stubs.values():
                stub.close()
            self._stubs.clear()
        return self.M.Ack()

    def UpdateGrad(self, request, context=None):          # core/Slave.scala:177-185
        if not self.is_async:
            raise RuntimeError("Cannot update gradient: slave is in synchronous mode.")
        delta = sparse_to_dense(request.gradUpdate, self.dim)
        nz = np.flatnonzero(delta)
        self.ctx.update_grad(nz.astype(np.int32), delta[nz])
        return self.M.Ack()


_METHODS = {  # method -> (request message, reply message)
    "RegisterSlave": ("Node", "Ack"), "UnregisterSlave": ("Node", "Ack"), "Forward": ("ForwardRequest", "ForwardReply"),
    "Gradient": ("GradientRequest", "GradUpdate"), "StartAsync": ("StartAsyncRequest", "Ack"),
    "StopAsync": ("Empty", "Ack"), "UpdateGrad": ("GradUpdate", "Ack"),
}


def serve_slave(servicer: SlaveServicer, port: int, host: str = "127.0.0.1", max_workers: int = 8):
    """`newServer(SlaveGrpc.bindService(new SlaveImpl, ec), node.port)` (core/Slave.scala:26; core/package.scala:16-17).
    A failing handler surfaces as a non-OK status (UNKNOWN), like an exception in the reference's Future.
    Returns (server, bound_port)."""
    import grpc
    M = servicer.M

    def wrap(fn):
        def handler(request, context):
            try:
                return fn(request, context)
            except Exception as e:  # failed Future -> Status.UNKNOWN with the message
                context.abort(grpc.StatusCode.UNKNOWN, f"{type(e).__name__}: {e}")
        return handler

    handlers = {}
    for name, (req, rep) in _METHODS.items():
        handlers[name] = grpc.unary_unary_rpc_method_handler(
            wrap(getattr(servicer, name)),
            request_deserializer=getattr(M, req).FromString,
            response_serializer=getattr(M, rep).SerializeToString)
    # The reference serves on a fixed 8-thread pool (utils/Pool.scala:13); the servicer serialises the request calls on its
    # device context with a lock, the async service calls (UpdateGrad, StopAsync) are safe while the loop runs.
    server = grpc.server(futures.ThreadPoolExecutor(max_workers=max_workers))
    server.add_generic_rpc_handlers((grpc.method_handlers_generic_handler(f"{PACKAGE}.Slave", handlers),))
    bound = server.add_insecure_port(f"{host}:{port}")    # usePlaintext (core/package.scala:20-21)
    server.start()
    return server, bound


class SlaveStub:
    """Client side of the same service (what the reference master's `SlaveGrpc.stub` is): used by the tests and
    usable to drive a real reference slave from Python."""

    def __init__(self, target: str):
        import grpc
        self.M = Messages()
        self.channel = grpc.insecure_channel(target)
        for name, (req, rep) in _METHODS.items():
            setattr(self, name, self.channel.unary_unary(
                f"/{PACKAGE}.Slave/{name}",
                request_serializer=getattr(self.M, req).SerializeToString,
                response_deserializer=getattr(self.M, rep).FromString))

    def close(self):
        self.channel.close()


_MASTER_METHODS = {"RegisterSlave": ("Node", "Ack"), "UnregisterSlave": ("Node", "Ack"), "UpdateGrad": ("GradUpdate", "Ack")}


class MasterStub:
    """Client side of service `epfl.distributed.Master` (proto.proto:13-19): what a slave holds as `masterStub`
    (core/Slave.scala:21-22) -- registration and, in async mode, the deltas (core/Slave.scala:105)."""

    def __init__(self, target: str):
        import grpc
        self.M = Messages()
        self.channel = grpc.insecure_channel(target)
        for name, (req, rep) in _MASTER_METHODS.items():
            setattr(self, name, self.channel.unary_unary(
                f"/{PACKAGE}.Master/{name}",
                request_serializer=getattr(self.M, req).SerializeToString,
                response_deserializer=getattr(self.M, rep).FromString))

    def close(self):
        self.channel.close()


def serve_master(handlers: Dict[str, Callable], port: int, host: str = "127.0.0.1", max_workers: int = 8):
    """A `Master` service endpoint with the given handlers (name -> fn(request) -> reply); methods without a handler answer
    Ack.  Enough for a Python-side master to receive registrations and async deltas from slaves (core/Master.scala:222-253;
    core/MasterAsync.scala:164-177).  Returns (server, bound_port)."""
    import grpc
    M = Messages()
    table = {}
    for name, (req, rep) in _MASTER_METHODS.items():
        fn = handlers.get(name, lambda request: M.Ack())

        def handler(request, context, fn=fn):
            try:
                out = fn(request)
                return out if out is not None else M.Ack()
            except Exception as e:
                context.abort(grpc.StatusCode.UNKNOWN, f"{type(e).__name__}: {e}")
        table[name] = grpc.unary_unary_rpc_method_handler(handler, request_deserializer=getattr(M, req).FromString,
                                                          response_serializer=getattr(M, rep).SerializeToString)
    server = grpc.server(futures.ThreadPoolExecutor(max_workers=max_workers))
    server.add_generic_rpc_handlers((grpc.method_handlers_generic_handler(f"{PACKAGE}.Master", table),))
    bound = server.add_insecure_port(f"{host}:{port}")
    server.start()
    return server, bound
