// A copy of `data` placed so that `pad` zero bytes after it end exactly at an inaccessible page: a decoder that reads
// further past its input than the library's padding allows faults.  run(buf) is called on the copy; returns what it
// returns, or -2 when the pages cannot be mapped.
#pragma once
#include <stdint.h>
#include <string.h>
#include <sys/mman.h>
#include <unistd.h>

template <class Run>
auto emu_guarded(const uint8_t* data, int64_t nbytes, int64_t pad, Run run) -> decltype(run(data)) {
    const int64_t page = sysconf(_SC_PAGESIZE);
    const int64_t body = (nbytes + pad + page - 1) / page * page;
    uint8_t* base = (uint8_t*)mmap(nullptr, body + page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (base == MAP_FAILED) return -2;
    mprotect(base + body, page, PROT_NONE);
    uint8_t* buf = base + body - pad - nbytes;
    memcpy(buf, data, (size_t)nbytes);
    memset(buf + nbytes, 0, (size_t)pad);
    const auto r = run(buf);
    munmap(base, body + page);
    return r;
}
