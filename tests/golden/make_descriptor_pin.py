"""Extracts the serialized FileDescriptorProto that protoc embedded in the reference's generated code
(examples/grpc-server/grpc/hello.pb.go: file_hello_proto_rawDesc) into tests/golden/hello_proto_rawdesc.hex.

It is the one byte string in the reference that a real protobuf encoder produced: tests/test_proto.py pins the proto3
encoder and decoder to it.  Needs a checkout of the reference (JigarJoshi04/gofr @ 17218229):

    python tests/golden/make_descriptor_pin.py <reference checkout>
"""
import os
import re
import sys

REF = os.path.join(sys.argv[1], "examples", "grpc-server", "grpc", "hello.pb.go")
HERE = os.path.dirname(os.path.abspath(__file__))

src = open(REF).read()
m = re.search(r"file_hello_proto_rawDesc = \[\]byte\{(.*?)\n\}", src, re.S)
raw = bytes(int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]{2})", m.group(1)))
with open(os.path.join(HERE, "hello_proto_rawdesc.hex"), "w") as f:
    f.write("# file_hello_proto_rawDesc of examples/grpc-server/grpc/hello.pb.go (%d bytes), see make_descriptor_pin.py\n" % len(raw))
    f.write(raw.hex() + "\n")
print(len(raw), "bytes")
