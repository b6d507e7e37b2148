# Builds the 3-D mask editor's CPU checker (test infrastructure; never linked into the product).
# Same flags as the other checkers: -ffp-contract=off, the reference (Rust) never fuses multiply-add.
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function

all: libeditor.so

libeditor.so: editor.c
	$(CC) $(CFLAGS) -o $@ editor.c -lm

clean:
	rm -f libeditor.so
