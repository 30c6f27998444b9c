"""TensorFlow GraphDef construction for the OpenCV tests, with the TF protos bundled in the `tensorboard` package.  The graphs run
in tests/opencv_tf_runner.py, a process of its own: OpenCV's protobuf runtime must not share a process with these protos."""
import subprocess
import sys

import numpy as np


def have_cv2():
    p = subprocess.run([sys.executable, "-c", "import cv2; print(hasattr(cv2.dnn, 'readNetFromTensorflow'))"], capture_output=True, text=True)
    return p.returncode == 0 and p.stdout.strip() == "True"


def protos():
    from tensorboard.compat.proto import graph_pb2, node_def_pb2, tensor_pb2, tensor_shape_pb2, types_pb2
    return graph_pb2, node_def_pb2, tensor_pb2, tensor_shape_pb2, types_pb2


def _shape(dims):
    _, _, _, ts, _ = protos()
    return ts.TensorShapeProto(dim=[ts.TensorShapeProto.Dim(size=int(d)) for d in dims])


def const(name, arr, integer=False):
    _, nd, tp, _, ty = protos()
    arr = np.asarray(arr)
    dt = ty.DT_INT32 if integer else ty.DT_FLOAT
    n = nd.NodeDef(name=name, op="Const")
    n.attr["dtype"].type = dt
    n.attr["value"].tensor.CopyFrom(tp.TensorProto(dtype=dt, tensor_shape=_shape(arr.shape),
                                                   tensor_content=arr.astype("<i4" if integer else "<f4").tobytes()))
    return n


def placeholder(name, shape):
    _, nd, _, _, ty = protos()
    n = nd.NodeDef(name=name, op="Placeholder")
    n.attr["dtype"].type = ty.DT_FLOAT
    n.attr["shape"].shape.CopyFrom(_shape(shape))
    return n


def node(name, op, inputs, **attrs):
    _, nd, _, _, ty = protos()
    n = nd.NodeDef(name=name, op=op, input=list(inputs))
    n.attr["T"].type = ty.DT_FLOAT
    for k, v in attrs.items():
        if isinstance(v, bytes):
            n.attr[k].s = v
        elif isinstance(v, bool):
            n.attr[k].b = v
        elif isinstance(v, float):
            n.attr[k].f = v
        elif isinstance(v, int):
            n.attr[k].i = v
        else:
            n.attr[k].list.i.extend(int(i) for i in v)
    return n
