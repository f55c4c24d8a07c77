"""A bad argument to a native op raises RuntimeError instead of killing the process.

A TORCH_CHECK message assembled from several arguments crashes this extension when it is thrown (the process dies with
SIGSEGV instead of raising), so every TORCH_CHECK under csrc/ takes at most one message argument.  The lint below
enforces that; the subprocess test checks that CPU ops given bad arguments raise with their message."""
import os
import re
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'graphlearn_for_pytorch_b200', 'csrc')

_CHECK = re.compile(r'\b(TORCH_CHECK|TORCH_INTERNAL_ASSERT)\s*\(')


def _strip_comments(src: str) -> str:
  """Blanks // and /* */ comments (string and char literals kept) so that line numbers stay put."""
  out, i, n = [], 0, len(src)
  while i < n:
    c = src[i]
    if c in '"\'':
      j = i + 1
      while j < n and src[j] != c:
        j += 2 if src[j] == '\\' else 1
      out.append(src[i:j + 1])
      i = j + 1
    elif src.startswith('//', i):
      j = src.find('\n', i)
      i = n if j < 0 else j
    elif src.startswith('/*', i):
      j = src.find('*/', i + 2)
      j = n if j < 0 else j + 2
      out.append(re.sub(r'[^\n]', ' ', src[i:j]))
      i = j
    else:
      out.append(c)
      i += 1
  return ''.join(out)


def _top_level_args(src: str, start: int):
  """Arguments of the call whose '(' is at src[start - 1]: top-level commas split them."""
  depth, i, cur, args = 0, start, [], []
  while i < len(src):
    c = src[i]
    if c in '"\'':
      j = i + 1
      while src[j] != c:
        j += 2 if src[j] == '\\' else 1
      cur.append(src[i:j + 1])
      i = j + 1
      continue
    if c in '([{':
      depth += 1
    elif c in ')]}':
      if depth == 0:
        args.append(''.join(cur).strip())
        return args
      depth -= 1
    elif c == ',' and depth == 0:
      args.append(''.join(cur).strip())
      cur = []
      i += 1
      continue
    cur.append(c)
    i += 1
  raise ValueError('unbalanced call')


def multi_part_checks(root: str = CSRC):
  """(file:line, macro) of every TORCH_CHECK / TORCH_INTERNAL_ASSERT with more than one message argument."""
  found = []
  for dirpath, _, files in os.walk(root):
    for f in sorted(files):
      if not f.endswith(('.cc', '.cu', '.h', '.cuh', '.cpp')):
        continue
      path = os.path.join(dirpath, f)
      with open(path) as fh:
        src = _strip_comments(fh.read())
      for m in _CHECK.finditer(src):
        args = _top_level_args(src, m.end())
        if len(args) > 2:
          line = src.count('\n', 0, m.start()) + 1
          found.append(f'{os.path.relpath(path, root)}:{line} {m.group(1)}')
  return found


def test_lint_parses_checks():
  # the parser sees through nested calls, templates, strings with commas and comments
  src = 'TORCH_CHECK(f(a, b) && g<int>(c), "x, y"); /* TORCH_CHECK(a, b, c) */ TORCH_CHECK(d, "e", f);'
  src = _strip_comments(src)
  calls = [_top_level_args(src, m.end()) for m in _CHECK.finditer(src)]
  assert calls == [['f(a, b) && g<int>(c)', '"x, y"'], ['d', '"e"', 'f']]


def test_every_check_has_one_message_argument():
  assert multi_part_checks() == []


_BAD_CALLS = textwrap.dedent(r'''
  import sys
  sys.path.insert(0, sys.argv[1])
  import torch
  import graphlearn_for_pytorch_b200 as glt
  nat = glt.ops.require_native()
  i64 = torch.arange(6, dtype=torch.int64)
  indptr = torch.tensor([0, 2, 4, 6], dtype=torch.int64)
  cases = [
    ('rows must be int64', lambda: nat.coo_to_csr(i64.int(), i64, None, None, 6, False)),
    ('indptr must be contiguous',
     lambda: nat.cpu_sample_neighbors(torch.arange(8, dtype=torch.int64)[::2], i64, None, i64[:2], 2, False, False,
                                      0, 0)),
    ('ids must be int64',
     lambda: nat.cpu_gather_rows(torch.zeros(6, 4), i64.int(), None, 0, torch.zeros(6, 4), None)),
  ]
  for msg, call in cases:
    try:
      call()
    except RuntimeError as e:
      assert msg in str(e), (msg, str(e))
      print('raised:', msg, flush=True)
    else:
      raise AssertionError(msg + ': did not raise')
''')


def test_cpu_ops_raise_on_bad_arguments(glt):
  # a subprocess, so that an op that crashes instead of raising fails this test without ending the test run
  r = subprocess.run([sys.executable, '-c', _BAD_CALLS, ROOT], capture_output=True, text=True, timeout=600)
  assert r.returncode == 0, f'exit code {r.returncode}\n{r.stdout}\n{r.stderr}'
  assert r.stdout.count('raised:') == 3, r.stdout
