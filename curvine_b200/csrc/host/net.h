// Blocking TCP helpers (the reference uses tokio sockets with TCP_NODELAY + keepalive:
// orpc/src/client/raw_client.rs:36-39, orpc/src/server/rpc_server.rs:179-181; sendfile loop sys_libc.rs:76-122).
#pragma once
#include "common.h"

namespace cv {

// conn_timeout_ms > 0: give up connecting after that long (raw_client.rs:51-55, client_conf.rs conn_timeout_ms);
// io_timeout_ms > 0: every send/recv on the socket fails with kIO "... timed out" after that long without progress
// (the blocking-socket stand-in for RpcClient::timeout_rpc(data_timeout_ms, ..), block_client.rs:56,88-95: an elapsed
// timer becomes io::ErrorKind::TimedOut, i.e. FsError::IO, orpc/src/io/io_error.rs:148-153)
Err tcp_connect(const std::string& host, int port, int* fd_out, int64_t conn_timeout_ms = 0, int64_t io_timeout_ms = 0);
Err tcp_listen(const std::string& host, int port, int* fd_out, int* bound_port);
// Same-host transport beside TCP (an addition of this project, no reference counterpart): the worker also listens on the ABSTRACT unix socket
// "curvine-b200-worker-<tcp port>" (no file system entry, same network namespace as the loopback port); a local client that is
// configured for it ([b200] local_unix_socket) connects there first.  Same frames, same handlers; unix
// sockets with sendfile carry more than loopback TCP at the same connection count (tools/loopback_probe.cc measures both).
std::string local_socket_name(int tcp_port);
Err unix_listen(const std::string& abstract_name, int* fd_out);
Err unix_connect(const std::string& abstract_name, int* fd_out, int64_t io_timeout_ms = 0);
// explicit SO_RCVBUF / SO_SNDBUF for sockets created from now on (0 = leave the kernel's autotuning alone, the default)
void set_socket_buffer_bytes(int bytes);
Err send_all(int fd, const void* buf, size_t n);
Err send_more(int fd, const void* buf, size_t n);  // MSG_MORE: more bytes of the same message follow at once
Err recv_exact(int fd, void* buf, size_t n);  // kIO "connection closed" on EOF
Err send_file_full(int sock, int file_fd, int64_t off, size_t n);
void set_sock_opts(int fd);
void close_fd(int fd);

}  // namespace cv
